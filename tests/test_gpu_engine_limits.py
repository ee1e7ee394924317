"""The engine at its documented limits on the pod-state plugins: 8 distinct topology keys (K), 12 topology counters per
dynamic class and 64 distinct host-port sets among pending pods (a uint64 mask).  At each limit every entry point that
derives the pending side answers bit for bit like the CPU oracle, which has no such limits; one step past it the call is
refused (status 1, "use the stock path") and the engine is left as it was.  The worlds come from limits_harness.py; a test
without the GPU shows, through a mirror of the host derivation, that they reach the limits and that the verdicts the
parity checks compare actually occur.  Seeds are fixed, and every failure names its seed."""
import copy
import random

import numpy as np
import pytest

import capacity_harness as CH
import group_reasons_ref as ref
import limits_harness as H
from delta_harness import _assert_same, _check, _oracle_results, _results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import capi
from kubernetes_autoscaler_b200 import drain as dr
from kubernetes_autoscaler_b200 import podlistprocessor as plp
from kubernetes_autoscaler_b200.encode import Encoder, RemovalPlan, encode
from kubernetes_autoscaler_b200.objects import (BuildTestPod, LabelSelector, NodeInfo, PodAffinityTerm, Requirement,
                                                TopologySpreadConstraint, makePodEquivalenceGroup)
from plan_harness import bytes_of_cluster, engine_plan, loop_plan, random_pdbs
from test_removal_batch import batch, oracle_loop

C = capi.CONST
SEEDS = [11, 12]


@pytest.fixture(scope="module")
def eng():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _encode(cluster, templates, groups):
    encoder = Encoder()
    return encoder, encode(cluster, templates, groups, encoder=encoder)


def _derive(cluster, templates, groups, enc, encoder):
    """limits_harness.derive with the EXIST activity judged on the objects"""
    name = {v: k for k, v in encoder.keys.ids.items()}
    rule = H.exist_rule(cluster, templates, [g.pods[0] for g in groups])
    off, pend = enc.arrays["group_off"], enc.arrays["pend_spec"]
    pod_of = {int(pend[off[g]]): groups[g].pods[0] for g in range(len(groups)) if off[g + 1] > off[g]}
    return H.derive(enc, lambda s, k: rule(pod_of[s], name[k]))


def _pods(groups):
    """Every pod of the groups as its own object (a group repeats one object), so that a pod order lists each pending pod
    once, as TrySchedulePods gets it"""
    out = []
    for g in groups:
        for k, p in enumerate(g.pods):
            q = p.clone()
            q.name = "%s-%d" % (p.name, k)
            out.append(q)
    return out


# ---- without the GPU: the inputs reach their cases ----------------------------------------------------------------------
def test_inputs_reach_the_limits():
    for seed in SEEDS:
        for host in (True, False):
            cl, tm, gr = H.world(seed, host=host)
            encoder, enc = _encode(cl, tm, gr)
            d = _derive(cl, tm, gr, enc, encoder)
            assert d["K"] == H.MAX_KEYS and any(d["is_host"]) == host, seed
            assert not host or d["is_host"].index(True) == 3, seed            # the hostname key away from slot 0
            full = [c for c in d["classes"].values() if len(c["kinds"]) == H.MAX_Q]
            assert len(full) >= 8 and max(len(c["kinds"]) for c in d["classes"].values()) == H.MAX_Q, seed
            assert {len(c["kinds"]) for c in d["classes"].values()} >= {8, 9, 10, 11, 12}, seed
            kinds = lambda c: [c["kinds"].count(q) for q in (H.Q_PTS, H.Q_AFF, H.Q_ANTI, H.Q_EXIST)]
            assert [2, 1, 1, 8] in [kinds(c) for c in full] and [4, 0, 0, 8] in [kinds(c) for c in full], seed
            assert any(not all(c["active"]) for c in full), seed                 # EXIST counters the ballot squeezes out
            assert any(all(c["active"]) for c in d["classes"].values()), seed
            names = {v: k for k, v in encoder.keys.ids.items()}
            dc = {names[k]: (d["Dc"][i], d["D"][i]) for i, k in enumerate(d["keys"])}
            assert dc["tmpl"][0] == 0 and dc["tmpl"][1] == 2, seed            # a key only templates carry
            assert dc["region"][1] > dc["region"][0], seed                     # template-only values
            assert dc["rack"] == (40, 45), seed
            assert d["n_port_sets"] == H.MAX_PORT_SETS, seed
        # compact ids 0 / 31 / 32 / 63 conflict pairwise across the word boundary, and not with their neighbours
        sets = H.port_sets()
        fam = [0, 31, 32, 63]
        for i in fam:
            for j in range(64):
                assert H.port_conflict(sets[i], sets[j]) == (j in fam), (i, j)
        ids = d["port_id"]
        a = enc.arrays
        first = sorted(ids, key=ids.get)
        for i in fam:                      # the list of compact id i is prototype i's
            pl = first[i]
            got = [(int(a["port_num"][x])) for x in range(a["port_off"][pl], a["port_off"][pl + 1])]
            assert sorted(got) == sorted(h.host_port for h in sets[i]), i
    # the large worlds: a non-hostname key with Dc past the 512-thread block
    for n in (513, 1100):
        cl, tm, gr = H.world(3, nodes=n)
        encoder, enc = _encode(cl, tm, gr)
        d = H.derive(enc)
        assert d["K"] == 8 and max(dc for dc, h in zip(d["Dc"], d["is_host"]) if not h) == n and d["is_host"].index(True) == 3
    # one step past each limit
    for what, check in (("key", lambda d: d["K"] == 9),
                        ("counter", lambda d: max(len(c["kinds"]) for c in d["classes"].values()) == 13),
                        ("port", lambda d: d["n_port_sets"] == 65)):
        protos = H.with_extra(H.pending_protos(11, H.KEYS), what)
        cl, tm, gr = H.world(11, protos=protos)
        encoder, enc = _encode(cl, tm, gr)
        d = H.derive(enc)
        assert check(d), what
        assert d["K"] <= 9 and d["n_port_sets"] <= 65
    # the movers of a removal batch: at the limits, and the 8th key brought by a mover alone
    cl = H.removal_world(11)
    _, enc = _encode(cl, [], [])
    after = _all_movers(enc)[3]
    d = H.derive(after)
    assert d["K"] == 8 and d["n_port_sets"] == 64 and max(len(c["kinds"]) for c in d["classes"].values()) == 12
    cl, _ = _mover_key_world(11, extra=False)
    _, enc = _encode(cl, [], [plp.build_pod_groups([BuildTestPod("x", 10, 10)])[0]])
    assert H.derive(enc)["K"] == 7 and H.derive(_all_movers(enc)[3])["K"] == 8
    cl, _ = _mover_key_world(11, extra=True)
    _, enc = _encode(cl, [], [plp.build_pod_groups([BuildTestPod("x", 10, 10)])[0]])
    assert H.derive(_all_movers(enc)[3])["K"] == 9


def test_oracle_verdicts_occur(oracle):
    """The parity checks are not vacuous: every pod-state verdict occurs on the oracle in the limit worlds, and a pod with
    port set 32 is refused by NodePorts on the node where a pod with set 31 was placed, and not without it."""
    seen = set()
    for seed in SEEDS:
        for host in (True, False):
            cl, tm, gr = H.world(seed, host=host)
            reasons, _ = oracle.feasibility_dense(encode(cl, tm, gr))
            seen |= set(np.unique(reasons).tolist())
    for code in ("CAE_R_PTS_SKEW", "CAE_R_PTS_MISSING_LABEL", "CAE_R_IPA_AFFINITY", "CAE_R_IPA_ANTI_AFFINITY",
                 "CAE_R_IPA_EXISTING_ANTI_AFFINITY", "CAE_R_OK"):
        assert C[code] in seen, code
    x, idx, ok = _ports_31_32(SEEDS[0])
    d = H.derive(x.enc)
    pl, pend = x.enc.arrays["ps_port_list"], x.enc.arrays["pend_spec"]
    assert [d["port_id"][int(pl[pend[i]])] for i in idx] == list(range(64))
    for order, want in _port_orders(idx):
        got = oracle.filter_schedulable(x.enc, order, None, None, None, ok, 0)[0]
        assert [int(got[i]) for i in order] == want, order


def _port_orders(idx):
    """(order, expected node of each pod) on the one acceptable row: set 32 is refused after set 31 and placed alone; sets
    32 apart that do not conflict (1 / 33, 30 / 62, 0 / 32 + 1 = 33) both land, so an id taken modulo 32 would show"""
    return [([idx[31], idx[32]], [0, -1]), ([idx[32]], [0]), ([idx[63], idx[0]], [0, -1]), ([idx[1], idx[33]], [0, 0]),
            ([idx[30], idx[62]], [0, 0]), ([idx[33], idx[1], idx[0]], [0, 0, 0])]


def _ports_31_32(seed):
    """The filter-pass inputs of the limit world with every pending pod plain apart from its ports, and only cluster row 0
    acceptable: (inputs, pending index of the pod with set i for every i, node filter)"""
    cl, _, gr = H.world(seed, templates=0)
    for ni in cl:
        ni.pods = [p for p in ni.pods if not p.pod_anti_affinity]
    pods = []
    for g in gr:
        p = g.pods[0].clone()
        p.topology_spread, p.pod_affinity, p.pod_anti_affinity = [], [], []
        p.requests = {"cpu": 1, "memory": 1}
        pods.append(p)
    x = plp.prepare_try_schedule(cl, pods)
    ok = np.zeros(len(cl), np.uint8)
    ok[0] = 1
    return x, list(x.order), ok


# ---- on the GPU: every entry point against its reference at the limits --------------------------------------------------
def _scale_up_parity(eng, oracle, enc, seed, caps=(0, 20, 300), light=False):
    from kubernetes_autoscaler_b200.engine import unpack_bits
    eng.load(enc)
    tag = "seed %d" % seed
    bits, reasons, count = eng.feasibility()
    want, _ = oracle.feasibility_dense(enc)
    assert np.array_equal(reasons, want), tag + " dense reasons"
    assert np.array_equal(unpack_bits(bits, enc.P), want == 0), tag + " dense bits"
    assert np.array_equal(count, (want == 0).sum(axis=1)), tag + " fit counts"
    assert np.array_equal(eng.feasibility_groups(), oracle.feasibility_groups(enc)), tag + " feasibility_groups"
    for cap in caps:
        c = np.full(enc.T, cap, np.int32)
        got = eng.estimate_all(c)
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, c)
        for g, w, nm in zip(got, (onc, opc, osched, oorder), ("nodes", "pods", "sched", "order")):
            assert np.array_equal(g, w), "%s cap %d: estimate %s differs" % (tag, cap, nm)
        mask, waste = eng.expander_best([0, 1, 2], got[0], got[1])
        omask, owaste = oracle.expander(enc, [0, 1, 2], onc, opc, osched)
        assert np.array_equal(mask, omask) and np.array_equal(waste, owaste), "%s cap %d expander" % (tag, cap)
        if light:
            continue
        assert np.array_equal(eng.waste_scores(), owaste), "%s cap %d waste" % (tag, cap)
        node_price = 1.0 + np.arange(enc.T) * 0.37
        pod_price = 0.01 + (np.arange(enc.struct.num_podspecs) % 13) * 0.003
        assert np.array_equal(eng.price_scores(node_price, pod_price, 0.5, 1500),
                              oracle.price_scores(enc, node_price, pod_price, 0.5, 1500, node_count=onc, sched=osched,
                                                  order=oorder)), "%s cap %d price" % (tag, cap)
    if light:
        return
    N = enc.struct.num_cluster_nodes
    li = (np.arange(enc.T, dtype=np.int32) * 37 + 3 * N + 5).astype(np.int32)       # raw: past the node list
    got = eng.estimate_all_li(np.full(enc.T, 25, np.int32), li)
    want = oracle.estimate_all_li(enc, np.full(enc.T, 25, np.int32), li)
    assert all(np.array_equal(g, w) for g, w in zip(got, want)), tag + " estimate_all_li"
    sched, counts, detail = eng.group_reasons(want_detail=True)
    ws, wc, wd = ref.group_reasons(enc)
    assert np.array_equal(detail, wd) and np.array_equal(sched, ws) and np.array_equal(counts, wc), tag + " group_reasons"


@pytest.mark.gpu
@pytest.mark.parametrize("host", [True, False], ids=["hostname", "no-hostname"])
def test_gpu_scale_up_entry_points(eng, oracle, host):
    for seed in SEEDS:
        cl, tm, gr = H.world(seed, host=host)
        _scale_up_parity(eng, oracle, encode(cl, tm, gr), seed)


@pytest.mark.gpu
@pytest.mark.parametrize("host", [True, False], ids=["hostname", "no-hostname"])
def test_gpu_filter_pass(eng, oracle, host):
    """filter_schedulable with hints, similarity classes and a node filter, ports and counters at the limits"""
    placed = {False: 0, True: 0}
    for seed in SEEDS:
        cl, _, gr = H.world(seed, templates=0, host=host)
        rng = random.Random(seed)
        pods = _pods(gr)
        rng.shuffle(pods)
        h = plp.Hints()
        for p in pods:
            if rng.random() < 0.15:
                h.Set((p.namespace, p.name), rng.choice(cl).node.name)
        banned = {ni.node.name for ni in cl if rng.random() < 0.15}
        x = plp.prepare_try_schedule(cl, pods, h, lambda ni: ni.node.name not in banned)
        assert sorted(x.order) == list(range(x.enc.P)), seed
        assert H.derive(x.enc)["n_port_sets"] == 64 and H.derive(x.enc)["K"] == 8, seed
        eng.load(x.enc)
        for li, brk in ((0, False), (3 * len(cl) + 7, False), (0, True), (5, True), (3 * len(cl) + 7, True)):
            want = oracle.filter_schedulable(x.enc, x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li, brk)
            got = eng.filter_schedulable(x.order, x.hint, x.sim_class, x.class_ctrl, x.node_ok, li, brk)
            assert np.array_equal(got[0], want[0]) and got[1:] == want[1:], "seed %d lastIndex %d break %s" % (seed, li, brk)
            placed[brk] += int((want[0] >= 0).sum())
            assert (want[0] < 0).any(), (seed, li, brk)
    assert placed[False] > 0 and placed[True] > 0, placed          # some breaks come after placements
    x, idx, ok = _ports_31_32(SEEDS[0])
    eng.load(x.enc)
    for order, _ in _port_orders(idx):
        for brk in (False, True):
            want = oracle.filter_schedulable(x.enc, order, None, None, None, ok, 0, brk)
            got = eng.filter_schedulable(order, None, None, None, ok, 0, brk)
            assert np.array_equal(got[0], want[0]) and got[1:] == want[1:], (order, brk)


def _removal_case(seed, host=True):
    cl = H.removal_world(seed, host=host)
    rng = random.Random(seed)
    names = [ni.node.name for ni in cl]
    cands = names + [rng.choice(names) for _ in range(4)] + ["not-a-node"]
    dest = {n: rng.random() < 0.9 for n in names}
    return cl, cands, dest


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_removal_batches(eng, oracle, persist):
    """simulate_removals (a removal load) and simulate_resident_removals, whose movers reach 64 port sets and 12 counters,
    against the oracle's loop of single removals"""
    from test_gpu_resident_removals import resident_batch
    for seed in SEEDS:
        for host in (True, False):
            cl, cands, dest = _removal_case(seed, host)
            want = oracle_loop(cl, cands, dest, persist, last_index=seed)
            assert batch(lambda: plp.HintingSimulator(eng), cl, cands, dest, persist, last_index=seed) == want, seed
            assert resident_batch(eng, cl, cands, dest, persist, last_index=seed) == want, seed
            assert {r[0] for r in want["results"]} == {"remove", "unremovable"}, seed


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_plan_removals(eng, oracle, persist):
    for seed in SEEDS:
        cl, cands, dest = _removal_case(seed)
        rng = random.Random(seed + 1)
        pdbs = random_pdbs(rng, cl, 12)
        by = bytes_of_cluster(cl)
        kw = dict(limit=rng.choice([-1, 30]), last_index=seed)
        got = engine_plan(eng, cl, cands, dest, persist, by, pdbs, **kw)
        assert got == loop_plan(cl, cands, dest, persist, by, pdbs, **kw), seed


@pytest.mark.gpu
def test_gpu_check_capacity(eng, oracle):
    """requests kept (booked) and reverted (checks that fail), over 64 port sets and 12-counter classes"""
    for seed in SEEDS:
        cl, _, gr = H.world(seed, templates=0)
        protos = [g.pods[0] for g in gr]
        booked = [CH.pr("bk", *[(p, 1) for p in protos[:8]])]
        reqs = [CH.pr("r%d" % i, *[(p, 1 + (i + j) % 2) for j, p in enumerate(protos[8 + 2 * i:10 + 2 * i])]) for i in range(28)]
        reqs.append(CH.pr("huge", (protos[5], 400)))
        want = CH.oracle_loop(cl, booked, reqs, last_index=seed)
        got = CH.run(plp.HintingSimulator(eng), cl, booked, reqs, True, last_index=seed)
        assert got == want, seed
        assert True in want["found"] and False in want["found"], seed


@pytest.mark.gpu
@pytest.mark.parametrize("nodes", [513, 1100])
def test_gpu_large_worlds(eng, oracle, nodes):
    """rack holds a value per cluster node: Dc past the 512-thread block and the counter stride past 1000; caps past 256"""
    cl, tm, gr = H.world(nodes, nodes=nodes, templates=4)
    enc = encode(cl, tm, gr)
    _scale_up_parity(eng, oracle, enc, nodes, caps=(300,), light=True)


@pytest.mark.gpu
def test_gpu_three_rank_estimate_shards_sum_to_one_engine(eng):
    from kubernetes_autoscaler_b200.engine import Engine
    cl, tm, gr = H.world(SEEDS[0], templates=7)
    enc = encode(cl, tm, gr)
    caps = np.full(enc.T, 20, np.int32)
    eng.load(enc)
    want = eng.estimate_all(caps)
    total = [np.zeros_like(w) for w in want]
    for rank in range(3):
        e = Engine(device=0, rank=rank, world_size=3)
        try:
            e.load(enc)
            got = e.estimate_all(caps)
            tb, te = e.template_shard(enc.T)
            for i, g in enumerate(got):
                total[i] = total[i] + np.where(g == -1, 0, g) if i == 3 else total[i] + g
                if i == 3:
                    assert np.array_equal(g[tb:te], want[3][tb:te]), "seed %d rank %d" % (SEEDS[0], rank)
        finally:
            e.close()
    for i in range(3):
        assert np.array_equal(total[i], want[i]), "seed %d output %d" % (SEEDS[0], i)


# ---- one step either side of each limit ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("what", ["key", "counter", "port"])
def test_gpu_load_and_pod_delta_refused_one_past(engines, oracle, what):
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    eng, fresh = engines(True)
    seed = SEEDS[0]
    protos = H.pending_protos(seed, H.KEYS)
    cl, tm, gr = H.world(seed, protos=H.with_extra(protos, what))
    with pytest.raises(EngineUnsupported):
        eng.load(encode(cl, tm, gr))
    cl, tm, gr = H.world(seed, protos=protos)
    encoder, enc = _encode(cl, tm, gr)
    eng.load(enc)
    before = _results(eng, enc)
    _assert_same(before, _oracle_results(oracle, enc, True), "seed %d at the limit" % seed)
    saved = copy.deepcopy(encoder)
    extra = H.with_extra(protos, what)[-1]
    delta = encoder.pod_delta(gr + [makePodEquivalenceGroup(extra, 2)])
    assert eng.load_pods(delta) == 1, "seed %d" % seed
    _assert_same(_results(eng, enc), before, "seed %d after the refused delta" % seed)
    # the engine still takes a delta at the limit (the groups regrouped) and answers as a fresh load and the oracle
    regrouped = gr[::-1]
    good = saved.pod_delta(regrouped)
    after = enc.apply_pod_delta(good)
    assert eng.load_pods(good, after) == 0, "seed %d" % seed
    _check_seed(seed, eng, fresh, oracle, after, True)


def _all_movers(enc):
    """Every resident of every cluster row as a candidate's movers: (cand, move_off, move_slot, objects after the call)"""
    N = enc.struct.num_cluster_nodes
    off = enc.arrays["node_pod_off"]
    cand = np.arange(N, dtype=np.int32)
    move_off = np.asarray(off[:N + 1] - off[0], np.int32)
    slots = np.concatenate([np.arange(off[r + 1] - off[r]) for r in range(N)]).astype(np.int32)
    return cand, move_off, slots, enc.apply_resident_removals(cand, move_off, slots)[0]


def _mover_key_world(seed, extra):
    """Residents' anti terms and the movers on 7 keys, and one mover spreading over the 8th (region); with `extra`, one
    more mover spreading over a 9th key.  Returns (cluster, row and slot of the 9th-key mover)"""
    keys = [k for k in H.KEYS if k != "region"]
    protos = H.pending_protos(seed, keys)
    p = BuildTestPod("q-region", 30, 1 << 24)
    p.labels = {"app": "e"}
    p.topology_spread = [TopologySpreadConstraint(1, "region", LabelSelector({"app": "e"}))]
    protos.append(p)
    if extra:
        protos = H.with_extra(protos, "key")
    cl = H.removal_world(seed, protos=protos)
    for ni in cl:
        for q in ni.pods:
            if q.name.startswith("rb-"):
                q.pod_anti_affinity = [t for t in q.pod_anti_affinity if t.topology_key != "region"]
    last = len(protos) - 1
    row = last % 40                        # removal_world: prototype i on node i % 40
    return cl, (row, next(i for i, q in enumerate(cl[row].pods) if q.name == "m%02d" % last))


def _past_removal_world(seed, what):
    """(cluster, row and slot of the mover that goes one past the limit)"""
    if what == "key":
        return _mover_key_world(seed, True)
    protos = H.with_extra(H.pending_protos(seed, H.KEYS), what)
    cl = H.removal_world(seed, protos=protos)
    last = len(protos) - 1
    row = last % 40                        # removal_world: prototype i on node i % 40
    return cl, (row, next(i for i, q in enumerate(cl[row].pods) if q.name == "m%02d" % last))


def _check_seed(seed, *a, **k):
    """delta_harness._check, its failure naming the seed"""
    try:
        return _check(*a, **k)
    except AssertionError as e:
        raise AssertionError("seed %d: %s" % (seed, e)) from None


def _dummy_group():
    return plp.build_pod_groups([BuildTestPod("x", 10, 10)])[0]


def _without(cand, move_off, slots, row, slot):
    keep, off = [], [0]
    for c in range(len(cand)):
        for s in slots[move_off[c]:move_off[c + 1]]:
            if not (cand[c] == row and s == slot):
                keep.append(int(s))
        off.append(len(keep))
    return np.asarray(off, np.int32), np.asarray(keep, np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["key", "counter", "port"])
def test_gpu_movers_one_past_the_limit_are_refused(engines, oracle, what):
    """cae_simulate_resident_removals and cae_plan_removals answer 1 when the movers bring the 9th key, the 13th counter or
    the 65th port set; nothing changes, and the same engine then answers the batch without that mover as a removal load
    of the objects after it does"""
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    eng, fresh = engines(False)
    seed = SEEDS[1]
    cl, (row, slot) = _past_removal_world(seed, what)
    _, enc = _encode(cl, [], [_dummy_group()])
    eng.load(enc)
    before = _results(eng, enc)
    cand, move_off, slots, _ = _all_movers(enc)
    rc = eng._simulate_resident_removals_raw(cand, move_off, slots, None, None, None, None, 0, False, 4096)[0]
    assert rc == 1, "seed %d %s" % (seed, what)
    _assert_same(_results(eng, enc), before, "seed %d after the refused resident batch" % seed)
    with pytest.raises(EngineUnsupported):
        eng.plan_removals(RemovalPlan(cand_node=cand, drain=np.full(int(move_off[-1]), dr.MOVE, np.uint8), unneeded_limit=-1,
                                      kube_system_ns=-1))
    _assert_same(_results(eng, enc), before, "seed %d after the refused plan" % seed)
    # without that mover: at the limit (8 keys, 12 counters, 64 sets), accepted
    off2, slots2 = _without(cand, move_off, slots, row, slot)
    after, pend, first = enc.apply_resident_removals(cand, off2, slots2)
    d = H.derive(after)
    at = {"key": d["K"], "counter": max(len(c["kinds"]) for c in d["classes"].values()), "port": d["n_port_sets"]}[what]
    assert at == {"key": 8, "counter": 12, "port": 64}[what], (seed, what, at)
    for persist in (False, True):
        eng.enc = enc
        if persist:
            eng.load(enc)
        got = eng.simulate_resident_removals(cand, off2, slots2, None, None, None, None, seed, persist, enc=after)
        fresh.load(after)
        res, li, log = fresh.simulate_removals(cand, off2, pend, None, None, None, None, seed, persist)
        log = log.copy()
        log[:, 1] = first[log[:, 1]]
        assert np.array_equal(got[0], res) and got[1] == li and np.array_equal(got[2], log), (seed, what, persist)
        eng.load(enc)


@pytest.mark.gpu
@pytest.mark.parametrize("persist", [False, True])
def test_gpu_movers_bring_the_eighth_key(eng, oracle, persist):
    """the 8th key arrives with a mover's spread constraint only: accepted, and equal to the oracle's loop"""
    from test_gpu_resident_removals import resident_batch
    cl, _ = _mover_key_world(SEEDS[0], False)
    names = [ni.node.name for ni in cl]
    dest = {n: True for n in names}
    want = oracle_loop(cl, names, dest, persist)
    assert resident_batch(eng, cl, names, dest, persist) == want, "seed %d" % SEEDS[0]
    by = bytes_of_cluster(cl)
    assert engine_plan(eng, cl, names, dest, persist, by) == loop_plan(cl, names, dest, persist, by), "seed %d" % SEEDS[0]


# ---- deltas at the limits --------------------------------------------------------------------------------------------------
def _new_cluster_node(i, cpu=4000):
    from limits_harness import _node
    lb = {H.HOST: "new%d" % i, H.ZONE: "z9", "pool": "p9", "rack": "nr%d" % i, "row": "w9", "tmpl": "T7", "sparse": "s7",
          "region": "north"}
    return NodeInfo(_node("new%d" % i, lb, cpu=cpu), [])


@pytest.mark.gpu
def test_gpu_delta_chain_at_the_limits(engines, oracle):
    """node churn (new values on every key); rows relabelled on rack, row and sparse (a label removed), which
    cae_load_nodes refuses with status 2 because it keeps the domains, and cae_load_node_churn applies as dirty rows; a
    cae_load_nodes step off the topology keys; a pod delta with a new 12-counter class; a template delta with new
    template-only values; then force-added pods with ports and anti-affinity.  After each step every entry point answers as
    a fresh load, and as the oracle after the node steps and the last"""
    eng, fresh = engines(True)
    seed = SEEDS[0]
    cl, tm, gr = H.world(seed)
    encoder, cur = _encode(cl, tm, gr)
    eng.load(cur)
    # 1. churn: two nodes leave, three join with new values on all eight keys
    cl = cl[2:] + [_new_cluster_node(i) for i in range(3)]
    churn = encoder.node_churn(cl)
    assert eng.load_node_churn(churn), "seed %d" % seed
    cur = cur.apply_node_churn(churn)
    _check_seed(seed, eng, fresh, oracle, cur, True)
    # 2. relabel rack, row and sparse on three rows: sparse removed from two, added to one
    rows = [r for r in range(len(cl)) if "sparse" in cl[r].node.labels][:2] + [r for r in range(len(cl)) if "sparse" not in cl[r].node.labels][:1]
    relabelled = list(cl)
    for r in rows:
        ni = copy.deepcopy(cl[r])
        ni.node.labels.update({"rack": "rr%d" % r, "row": "w%d" % (r % 2)})
        if ni.node.labels.pop("sparse", None) is None:
            ni.node.labels["sparse"] = "s1"
        relabelled[r] = ni
    assert len(rows) == 3, seed
    before = _results(eng, cur)
    saved = copy.deepcopy(encoder)
    assert eng.load_nodes(encoder.node_delta([(r, relabelled[r]) for r in rows])) is False, seed
    _assert_same(_results(eng, cur), before, "seed %d after the refused node delta" % seed)
    encoder, cl = saved, relabelled
    churn = encoder.node_churn(cl)
    assert len(churn.arrays["removed"]) == 0 and len(churn.arrays["name"]) == 0
    assert eng.load_node_churn(churn), "seed %d" % seed
    cur = cur.apply_node_churn(churn)
    _check_seed(seed, eng, fresh, oracle, cur, True)
    # 2b. cae_load_nodes on rows whose topology labels stay: a new label off the keys, new allocatable
    changed = []
    for r in (2, 9):
        ni = copy.deepcopy(cl[r])
        ni.node.labels["gen"] = "g%d" % r
        ni.node.allocatable["cpu"] += 500
        cl[r] = ni
        changed.append((r, ni))
    nd = encoder.node_delta(changed)
    assert eng.load_nodes(nd), seed
    cur = cur.apply_node_delta(nd)
    _check_seed(seed, eng, fresh, oracle, cur, True, with_oracle=False)
    # 3. a new class with exactly 12 counters (2 PTS + 1 AFF + 1 ANTI + 8 EXIST), some groups leave
    p = BuildTestPod("twelve", 120, 1 << 26)
    p.labels = {"app": "a", "v": "2"}
    p.topology_spread = [TopologySpreadConstraint(1, "rack", LabelSelector({"app": "a"})),
                         TopologySpreadConstraint(2, "region", LabelSelector(match_expressions=[Requirement("app", "In", ["a", "b"])]),
                                                  min_domains=3)]
    p.pod_affinity = [PodAffinityTerm(LabelSelector({"app": "ra"}), "pool")]
    p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": "a"}), "tmpl")]
    gr = gr[3:] + [makePodEquivalenceGroup(p, 4)]
    pd = encoder.pod_delta(gr)
    cur = cur.apply_pod_delta(pd)
    assert eng.load_pods(pd, cur) == 0, "seed %d" % seed
    assert H.MAX_Q in {len(c["kinds"]) for c in H.derive(cur)["classes"].values()}, "seed %d" % seed
    _check_seed(seed, eng, fresh, oracle, cur, True, with_oracle=False)
    # 4. a template with new template-only values joins, one changes
    t5 = copy.deepcopy(tm[1])
    t5.node.name = "t5"
    t5.node.labels.update({H.HOST: "t5", "rack": "tr55", "tmpl": "T5", "region": "venus", "sparse": "s8"})
    tm2 = copy.deepcopy(tm)
    tm2[2].node.labels["region"] = "pluto"
    td = encoder.template_delta(tm2 + [t5])
    cur = cur.apply_template_delta(td)
    assert eng.load_templates(td, cur), "seed %d" % seed
    _check_seed(seed, eng, fresh, oracle, cur, True, with_oracle=False)
    # 5. force-add pending pods with ports and anti-affinity onto distinct rows
    off = cur.arrays["group_off"]
    idx = [int(off[g]) for g, grp in enumerate(gr) if grp.pods[0].host_ports and grp.pods[0].pod_anti_affinity][:6]
    assert len(idx) >= 3, "seed %d" % seed
    rows = [3 * k + 1 for k in range(len(idx))]
    cur, _ = cur.apply_force_add(idx, rows)
    assert eng.force_add_pods(idx, rows, cur) is not False, "seed %d" % seed
    _check_seed(seed, eng, fresh, oracle, cur, True)


# ---- the estimator's placement log ------------------------------------------------------------------------------------------
def log_world(n_pods, nodes=40):
    """Two groups of small pods that feed each other's spread counters (rack: a value per node) and an affinity group, on
    ~40 cluster nodes and one roomy template; every placement is logged."""
    rng = random.Random(n_pods)
    cl = [NodeInfo(H._node("c%02d" % i, H.cluster_labels(i, rng, H.KEYS), cpu=200, pods=3), []) for i in range(nodes)]
    tm = [NodeInfo(H._node("t0", H.template_labels(0, H.KEYS), cpu=64000, mem=256 << 30, pods=250), [])]
    groups = []
    for app, other in (("x", "y"), ("y", "x")):
        p = BuildTestPod("log-" + app, 10, 1 << 20)
        p.labels = {"app": app}
        sel = LabelSelector(match_expressions=[Requirement("app", "In", [app, other])])
        p.topology_spread = [TopologySpreadConstraint(10 ** 6, "rack", sel), TopologySpreadConstraint(1, "row", sel,
                                                                                                   when_unsatisfiable="ScheduleAnyway")]
        groups.append(makePodEquivalenceGroup(p, n_pods))
    return cl, tm, groups


# log_world(n) is drawn from seed n.  Measured on an H100: 1 258 pods per group fit the log (4 * (N + cap) + 1024 = 1 264
# entries here), 1 259 are the fewest that overflow it
LOG_FITS, LOG_OVERFLOWS = 1258, 3000


@pytest.mark.gpu
def test_gpu_placement_log_capacity(eng, oracle):
    """Just below the log's capacity the estimate equals the oracle; well past it the call answers status 1, not a result, and
    the next call on the same engine equals the oracle."""
    from kubernetes_autoscaler_b200.engine import EngineUnsupported
    caps = np.full(1, 20, np.int32)
    small = encode(*log_world(LOG_FITS))
    eng.load(small)
    got = eng.estimate_all(caps)
    want = oracle.estimate_all(small, caps)[:4]
    assert all(np.array_equal(g, w) for g, w in zip(got, want)), "seed %d" % LOG_FITS
    for n in (LOG_FITS + 1, LOG_OVERFLOWS):
        big = encode(*log_world(n))
        eng.load(big)
        with pytest.raises(EngineUnsupported):
            eng.estimate_all(caps)
        want = oracle.estimate_all(big, np.full(1, 1, np.int32))[:4]
        got = eng.estimate_all(np.full(1, 1, np.int32))
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), "seed %d: the call after the overflow" % n
