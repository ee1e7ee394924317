"""No answer depends on the calls made before it.  Every read-only entry point (tests/call_order.py) is made in random
orders on one engine, and each answer is compared bit for bit with a new engine that loads the same snapshot and makes
only that call; each (snapshot, call) is also checked once against the oracle or a host mirror.  Targeted cases: the
last estimate's device rows survive every other call; the group-reason cache after each state-changing call; the
estimator slab across layouts (window / slab, counter stride, active dims, block count) and across data in one layout;
the filter pass, removal batch and capacity batch sharing their one-block buffers; two engines in one process.  The
non-GPU tests classify every entry point of the header and show the generators reach every call and layout."""
import os

import numpy as np
import pytest

import call_order as co
import rank_layout
from delta_harness import _gen
from kubernetes_autoscaler_b200 import capi, synth

DEFAULT_BLOCKS = 3
BLOCKS = int(os.environ.get("CAE_ORDER_FUZZ_BLOCKS", str(DEFAULT_BLOCKS)))   # SEQUENCES random sequences each
SEQUENCES = 4


@pytest.fixture(scope="module")
def engs():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    a, b = Engine(device=0, want_reasons=True), Engine(device=0, want_reasons=True)
    yield a, b
    a.close()
    b.close()


@pytest.fixture(scope="module")
def ref(oracle):
    return co.Reference(oracle)


class Runner:
    """One engine under test: its snapshot, its last estimate and the calls made so far (for the failure message)."""

    def __init__(self, eng, ref, label):
        self.eng, self.ref, self.label = eng, ref, label
        self.snap, self.est, self.calls = None, None, []

    def load(self, snap):
        self.eng.load(snap.enc)
        self.snap, self.est = snap, None
        self.calls.append("load %s" % (snap.sid,))

    def call(self, name, args):
        kind = co.CATALOGUE[name].kind
        assert kind != "consumer" or self.est is not None
        got = co.answer(self.eng, self.snap.enc, name, args)
        self.calls.append(name)
        co.check_status(name, got)
        want = self.ref.want(self.snap, name, args, self.est)
        assert co.same(got, want), "%s, step %d: %s differs from a single-call engine; calls so far: %s" % (
            self.label, len(self.calls) - 1, name, " -> ".join(self.calls))
        if kind == "estimate":
            self.est = None if co.refused(got) else (name, args)
        return got


def _run_plan(runner, snaps, steps):
    for op, i, args in steps:
        if op == "load":
            runner.load(snaps[i])
        elif co.CATALOGUE[op].kind != "consumer" or runner.est is not None:   # (an estimate that overflowed its log)
            runner.call(op, args)


# ---- 2. random sequences ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("block", range(BLOCKS))
def test_random_sequences(engs, ref, block):
    snaps = co.block_snaps(block)      # every one loads: the plans below are the ones the non-GPU test inspects
    for s in range(SEQUENCES):
        seed = 1000 * block + s
        _run_plan(Runner(engs[0], ref, "seed %d" % seed), snaps, co.plan(seed, snaps))


# ---- 3a. the last estimate survives every other call ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("est", ["estimate_all", "estimate_all_ex"])
def test_estimate_survives_every_call(engs, ref, est):
    rng = np.random.default_rng(7)
    for snap in (co.synth_snap("c4"), co.slab_snap(3), co.world_snap(41_002, overfull=True, big=True)):
        r = Runner(engs[0], ref, "%s on %s" % (est, snap.sid))
        r.load(snap)
        r.call(est, co.CATALOGUE[est].gen(rng, snap.enc))
        consumers = [(n, co.CATALOGUE[n].gen(rng, snap.enc)) for n in co.CONSUMERS]
        first = [r.call(n, a) for n, a in consumers]
        for name in co.PLAIN:
            if co.CATALOGUE[name].kind == "estimate":
                continue
            r.call(name, co.CATALOGUE[name].gen(rng, snap.enc))
            for (n, a), was in zip(consumers, first):
                assert co.same(r.call(n, a), was), "%s changed after %s" % (n, name)


# ---- 3b. the group-reason cache after each state-changing call ------------------------------------------------------------
def _warm(eng, enc):
    eng.enc = enc
    eng.feasibility_groups()
    eng.estimate_all(np.full(enc.T, 40, np.int32))


def _ch_pending(eng, cur, seed):
    """the groups in reverse order: each group index now names another spec (a snapshot without counters takes that)"""
    pending = co.reversed_groups(cur)
    assert eng.load_pending(pending)
    return pending


def _ch_nodes(eng, cur, seed):
    delta, pending = synth.node_churn(cur, seed, 4)
    assert eng.load_pending(pending)
    _warm(eng, pending)
    assert eng.load_nodes(delta)
    return pending.apply_node_delta(delta)


def _ch_churn(eng, cur, seed):
    churn, pending = synth.node_scale(cur, seed, 1, 2, 3)
    assert eng.load_pending(pending)
    _warm(eng, pending)
    assert eng.load_node_churn(churn)
    return pending.apply_node_churn(churn)


def _ch_upcoming(eng, cur, seed):
    from test_gpu_upcoming_nodes import _copies
    up = _copies(cur, [seed % cur.T, 0, 0])
    assert eng.add_upcoming_nodes(up)
    return cur.apply_upcoming(up)


def _ch_templates(eng, cur, seed):
    delta = synth.template_churn(cur, seed, 2, 1, 2)
    after = cur.apply_template_delta(delta)
    assert eng.load_templates(delta, after)
    return after


def _ch_pods(eng, cur, seed):
    delta = synth.pod_churn(cur, seed, 2, 1)
    after = cur.apply_pod_delta(delta)
    assert eng.load_pods(delta, after) == 0
    return after


def _ch_force_add(eng, cur, seed):
    go, N = cur.arrays["group_off"], cur.struct.num_cluster_nodes
    pods = np.arange(go[1], go[2])        # every pod of group 1: the group is emptied
    nodes = (np.arange(len(pods)) + seed) % max(N, 1)
    after, _ = cur.apply_force_add(pods, nodes)
    assert eng.force_add_pods(pods, nodes, after) is not False
    return after


def _ch_daemonsets(eng, cur, seed):
    from kubernetes_autoscaler_b200.daemonset import pack_rows
    from test_gpu_template_daemonsets import _apply_case
    ds, ev, run, keep = _apply_case(cur, seed)
    eng.template_daemonsets(ds, ev, pack_rows(run, len(ds)), keep)
    return eng.enc


def _ch_resident_removals(eng, cur, seed):
    from test_gpu_resident_removals import _random_lists
    cand, off, slots, _ = _random_lists(cur, seed)
    after = cur.apply_resident_removals(cand, off, slots)[0]
    eng.simulate_resident_removals(cand, off, slots, persist=True, enc=after)
    return after


def _ch_plan_removals(eng, cur, seed):
    from test_gpu_removal_plan import _random_plan
    eng.plan_removals(_random_plan(cur, seed, True))
    return eng.enc


CHANGES = {"load_pending": _ch_pending, "load_nodes": _ch_nodes, "load_node_churn": _ch_churn,
           "add_upcoming_nodes": _ch_upcoming, "load_templates": _ch_templates, "load_pods": _ch_pods,
           "force_add_pods": _ch_force_add, "template_daemonsets (apply)": _ch_daemonsets,
           "simulate_resident_removals": _ch_resident_removals, "plan_removals": _ch_plan_removals}


@pytest.mark.gpu
@pytest.mark.parametrize("change", sorted(CHANGES))
def test_cache_after_each_state_change(engs, ref, change):
    """warm the cache (feasibility_groups, an estimate), make the change, then ask a cache reader first: equal to a fresh
    load of the objects after the change"""
    eng = engs[0]
    cur = _gen("c2" if change == "load_pending" else "c4")
    for k, first in enumerate(["estimate_all", "group_reasons", "similar_node_groups"]):
        eng.load(cur)
        _warm(eng, cur)
        after = CHANGES[change](eng, cur, 900 + k)
        snap = co.Snap(("after", change, k), after)
        r = Runner(eng, ref, "after %s" % change)
        r.snap = snap
        r.call(first, co.CATALOGUE[first].gen(np.random.default_rng(k), after))


# ---- 3c. the estimator slab across layouts --------------------------------------------------------------------------------
def _layouts():
    """name -> (snapshot, caps, its other-data twin).  window / slab: cap 40 against 0 with P above the window; host_*: a
    hostname counter, whose stride follows the cap; the slab at other active dims and at 10x the templates (blocks).  The
    host_* snapshots have counters, so their launches read the slot versions; a twin is the snapshot with its groups
    reversed, which keeps every input of the slab's layout signature (A, the node counts, P, the counters' domains) and
    so the slab, versions included, is not zeroed between the two."""
    A, P = 3, rank_layout.window_nodes(3) + 64
    host, slab = co.host_spread_snap(P), co.slab_snap(A)
    out = {"window": (slab, 40), "slab": (slab, 0), "host_cap5": (host, 5), "host_cap40": (host, 40), "host_slab": (host, 0),
           "slab_A5": (co.slab_snap(5), 0), "slab_T40": (co.slab_snap(A, templates=40), 0)}
    return {name: (snap, cap, co.twin(snap)) for name, (snap, cap) in out.items()}


LAYOUT_PAIRS = [("window", "slab"), ("host_cap5", "host_cap40"), ("host_slab", "host_cap40"), ("slab", "slab_A5"),
                ("slab", "slab_T40"), ("slab_A5", "window")]


@pytest.mark.gpu
def test_estimator_slab_across_layouts(engs, ref):
    layouts = _layouts()
    r = Runner(engs[0], ref, "slab layouts")

    def estimate(snap, cap):
        if r.snap is not snap:
            r.load(snap)
        r.call("estimate_all", dict(caps=np.full(snap.enc.T, cap, np.int32)))
        r.call("waste_scores", {})

    for x, y in LAYOUT_PAIRS:            # X, Y, X
        for name in (x, y, x):
            snap, cap, _ = layouts[name]
            estimate(snap, cap)
    for name, (snap, cap, twin) in sorted(layouts.items()):   # X, X': the same layout, other data
        estimate(snap, cap)
        estimate(twin, cap)
        estimate(snap, cap)


# ---- 3d. the one-block passes' shared buffers -----------------------------------------------------------------------------
@pytest.mark.gpu
def test_one_block_buffers_alternate(engs, ref):
    rng = np.random.default_rng(3)
    for snap in (co.world_snap(41_010, big=True), co.synth_snap("c3")):
        r = Runner(engs[0], ref, "one-block buffers on %s" % (snap.sid,))
        r.load(snap)
        P = snap.enc.P
        gens = {"filter_schedulable": lambda n: co.g_filter(rng, snap.enc, n),
                "simulate_removals": lambda n: co.g_removals(rng, snap.enc, n),
                "check_capacity": lambda n: co.g_capacity(rng, snap.enc, n)}
        for sizes in ([P] * 7, [P // 3, P, P // 2, 5, P, P // 4, 1]):   # every pass with n_pods == P, then other sizes
            for k, n in enumerate(sizes):
                name = ["filter_schedulable", "simulate_removals", "check_capacity"][k % 3 if k < 3 else (k * 2) % 3]
                r.call(name, gens[name](n))


# ---- 3e. two engines on one device ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_engines_alternate(engs, ref):
    snaps = co.block_snaps(1)
    runners = [Runner(engs[0], ref, "engine 0"), Runner(engs[1], ref, "engine 1")]
    plans = [co.plan(500, snaps, steps=24), co.plan(501, snaps, steps=24)]
    for k in range(max(map(len, plans))):
        for r, p in zip(runners, plans):
            if k < len(p):
                _run_plan(r, snaps, [p[k]])


# ---- 4. without a GPU -----------------------------------------------------------------------------------------------------
STATE_CHANGING = {
    "cae_load": "replaces the resident snapshot",
    "cae_load_pending": "replaces the pending pods",
    "cae_load_nodes": "rewrites cluster-node rows",
    "cae_load_node_churn": "adds and removes cluster nodes",
    "cae_add_upcoming_nodes": "adds copies of templates as cluster nodes",
    "cae_load_templates": "changes, adds and removes templates",
    "cae_load_pods": "appends pod specs and replaces the pending pods",
    "cae_force_add_pods": "moves pending pods onto cluster rows",
    "cae_simulate_resident_removals": "makes the movers the pending pods",
    "cae_plan_removals": "makes the potential movers the pending pods",
}
HOST_ONLY = {
    "cae_create": "makes an engine", "cae_destroy": "frees an engine", "cae_last_error": "the thread's last message",
    "cae_version": "a constant string", "cae_expander_chain": "host filter chain, reads no engine",
    "cae_expander_chain_ex": "host filter chain, reads no engine", "cae_get_stats": "counters of the host side",
    "cae_device_buffer": "a device pointer, no answer", "cae_stream": "the engine's stream handle",
    "cae_peer_handle": "multi-GPU plumbing", "cae_peer_attach": "multi-GPU plumbing",
    "cae_host_alloc": "pinned host memory", "cae_host_free": "pinned host memory",
}


def test_every_entry_point_is_classified():
    """a new entry point fails here until it is in the catalogue or listed as state-changing or host-only
    (cae_template_daemonsets is both: the catalogue makes it without apply)"""
    covered = {c.fn for c in co.CATALOGUE.values()}
    declared = set(capi.declared_functions())
    assert not covered & set(HOST_ONLY) and not covered & set(STATE_CHANGING)
    assert covered | set(STATE_CHANGING) | set(HOST_ONLY) == declared, sorted(declared ^ (covered | set(STATE_CHANGING) | set(HOST_ONLY)))


def test_generators_reach_every_call_and_layout():
    """the default sequences make every catalogue call, each block loads a snapshot whose uncapped estimate takes the slab,
    the layout pairs of the slab test differ in what they are named for, and each twin keeps its snapshot's layout"""
    seen = set()
    for block in range(DEFAULT_BLOCKS):    # a block's plans do not depend on how many blocks run
        snaps = co.block_snaps(block)
        assert any(not rank_layout.uses_window(rank_layout.layout_of(s.enc)["A"], s.enc.P, [0] * s.enc.T) for s in snaps), block
        for s in range(SEQUENCES):
            seen |= {op for op, _, _ in co.plan(1000 * block + s, snaps)}
    assert set(co.CATALOGUE) <= seen, sorted(set(co.CATALOGUE) - seen)
    lay = _layouts()

    def sig(name):
        snap, cap, _ = lay[name]
        A = rank_layout.layout_of(snap.enc)["A"]
        return dict(window=rank_layout.uses_window(A, snap.enc.P, [cap] * snap.enc.T), A=A, T=snap.enc.T,
                    host=co.has_host_counter(snap.enc), cap=cap)

    assert sig("window")["window"] and not sig("slab")["window"] and not sig("host_slab")["window"]
    assert sig("host_cap5")["host"] and sig("host_cap5")["cap"] != sig("host_cap40")["cap"]
    assert sig("slab_A5")["A"] != sig("slab")["A"] and sig("slab_T40")["T"] >= 10 * sig("slab")["T"]
    assert all(sig(n)["host"] for n in ("host_cap5", "host_cap40", "host_slab"))
    for name, (snap, cap, twin) in lay.items():   # the twins keep every table but the pending order, and change the data
        x, y = snap.enc.arrays, twin.enc.arrays
        assert set(x) == set(y) and (snap.enc.P, snap.enc.T, snap.enc.E) == (twin.enc.P, twin.enc.T, twin.enc.E), name
        assert all(np.array_equal(x[k], y[k]) for k in x if k not in ("pend_spec", "group_off")), name
        assert rank_layout.layout_of(snap.enc) == rank_layout.layout_of(twin.enc), name
        assert not np.array_equal(x["pend_spec"], y["pend_spec"]), name
    for x, y in LAYOUT_PAIRS:
        assert sig(x) != sig(y), (x, y)
