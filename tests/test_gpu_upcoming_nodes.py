"""cae_add_upcoming_nodes on the GPU: after a scale-up's upcoming nodes are added as copies of their templates (alone or with
the loop's node churn in the same call) every entry point answers bit-identically to a second engine freshly loaded with
EncodedObjects.apply_upcoming(...), and to the oracle where that is affordable — dense bits / reasons / counts, group
reasons, Estimate() (capped, unlimited, RAW lastIndex), waste and price scores, the filter-out-schedulable pass.  A pending
pod that fits only an upcoming copy is placed there by the filter pass and, force-added, no longer asks for a node.
Loop sequences (copies replaced by the registered node in the next call, chained loops interleaved with the other
deltas), empty and T = 0 calls, and every refusal (status 2) and malformed input (status -2) with the engine left as it
was."""
import numpy as np
import pytest

from delta_harness import _assert_same, _check, _gen, _results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import NodeChurn, NodeDelta, UpcomingNodes
from kubernetes_autoscaler_b200.objects import (LABEL_HOSTNAME, BuildTestPod, HostPort, LabelSelector, NodeInfo, PodAffinityTerm,
                                                PodEquivalenceGroup, TopologySpreadConstraint, WithLabels, WithNamespace,
                                                WithPodAntiAffinity)
from kubernetes_autoscaler_b200.upcoming import sanitized_node_info, upcoming_node_infos

from test_node_delta_host import _encoder, _node
from test_upcoming_nodes_host import _ds_pod

pytestmark = pytest.mark.gpu


def _labels(enc, ls):
    a = enc.arrays
    return dict(zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist(), a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist()))


def _copies(cur, tmpl, churn=None, new_zone=()):
    """UpcomingNodes of copies of templates `tmpl` of `cur` (the objects the engine holds), with `churn` in the same call:
    each copy's label set is its template's with a new hostname value; the copies listed in `new_zone` also take one new
    zone value.  The value and label-set tails continue those of the churn's `changed`."""
    a, s = cur.arrays, cur.struct
    N = s.num_cluster_nodes
    ch = churn.changed if churn is not None else None
    nv0 = s.num_values + (ch.struct.num_new_values if ch is not None else 0)
    nl0 = s.num_labelsets + (ch.struct.num_new_labelsets if ch is not None else 0)
    pairs = []
    for j, t in enumerate(tmpl):
        lab = _labels(cur, int(a["node_labelset"][N + t]))
        lab[synth.K_HOST] = nv0 + j
        if j in new_zone:
            lab[synth.K_ZONE] = nv0 + len(tmpl)
        pairs.append(sorted(lab.items()))
    nv = len(tmpl) + (1 if len(new_zone) else 0)
    ca = ch.arrays if ch is not None else {"value_is_int": [], "value_int": [], "ls_off": [0], "ls_key": [], "ls_val": []}
    lo = np.asarray(ca["ls_off"], np.int64)
    tails = dict(value_is_int=np.concatenate([ca["value_is_int"], np.zeros(nv)]),
                 value_int=np.concatenate([ca["value_int"], np.zeros(nv)]),
                 ls_off=np.concatenate([lo, lo[-1] + np.cumsum([len(p) for p in pairs], dtype=np.int64)]),
                 ls_key=np.concatenate([ca["ls_key"], [k for p in pairs for k, _ in p]]),
                 ls_val=np.concatenate([ca["ls_val"], [v for p in pairs for _, v in p]]))
    changed = ch.replace(**tails) if ch is not None else NodeDelta(**tails)
    churn = churn.replace(changed=changed) if churn is not None else NodeChurn(changed)
    name0 = int(max(a["node_name"].max(initial=0), np.max(churn.arrays["name"], initial=0))) + 1000
    return UpcomingNodes(churn, template_idx=list(tmpl), name=[name0 + j for j in range(len(tmpl))],
                         labelset=[nl0 + j for j in range(len(tmpl))])


KINDS = {"copies": ((0, 0, 3, -1), (), None), "new zone": ((1, 2, 2), (0, 2), None), "with churn": ((0, 4, -1), (1,), (4, 7, 5))}


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
@pytest.mark.parametrize("shape", ["c2", "c3", "c4"])
def test_upcoming_matches_full_load(engines, oracle, shape, want_reasons):
    eng, fresh = engines(want_reasons)
    enc = _gen(shape)
    for k, (kind, (tmpl, zone, scale)) in enumerate(sorted(KINDS.items())):
        tmpl = [t % enc.T for t in tmpl]
        churn, pending = synth.node_scale(enc, 31 + k, *scale) if scale else (None, enc)
        up = _copies(enc, tmpl, churn, zone)
        after = pending.apply_upcoming(up)
        assert after.struct.num_cluster_nodes == enc.struct.num_cluster_nodes + len(tmpl) + \
            (churn.num_added - churn.num_removed if churn is not None else 0)
        eng.load(enc)
        assert eng.add_upcoming_nodes(up), kind
        if pending is not enc:
            assert eng.load_pending(pending)
        _check(eng, fresh, oracle, after, want_reasons, with_oracle=want_reasons)


def _provisioned_world():
    """Two full cluster nodes, templates with DaemonSet pods (t0 roomy; t1 with a DaemonSet host port; t2 at its pod limit
    with its one DaemonSet pod), and pending pods that fit only a new node: plain ones, one with the DaemonSet's host port,
    one with anti-affinity to the DaemonSet pods' label, and hostname-spread ones."""
    ds_port = _ds_pod("ds-port")
    ds_port.host_ports = [HostPort(9100)]
    ds_port.labels["role"] = "agent"
    full = [NodeInfo(_node("n%d" % i, "z0", "a", cpu=100, pods=20), []) for i in range(2)]
    templates = [NodeInfo(_node("t0", "z0", "a", cpu=4000, pods=30), [_ds_pod("ds-a"), _ds_pod("ds-b", 300)]),
                 NodeInfo(_node("t1", "z1", "b", cpu=4000, pods=30), [ds_port]),
                 NodeInfo(_node("t2", "z9", "a", cpu=8000, pods=1), [_ds_pod("ds-a")])]
    for ni in templates:
        for p in ni.pods:
            p.node_name = ni.node.name
    plain = BuildTestPod("work", 1000, 256 << 20, WithNamespace("ns1"), WithLabels({"app": "work"}))
    port = BuildTestPod("porty", 200, 64 << 20, WithNamespace("ns1"), WithLabels({"app": "porty"}))
    port.host_ports = [HostPort(9100)]
    shy = BuildTestPod("shy", 200, 64 << 20, WithNamespace("ns1"), WithLabels({"app": "shy"}),
                       WithPodAntiAffinity(PodAffinityTerm(LabelSelector(match_labels={"role": "agent"}), LABEL_HOSTNAME)))
    spread = BuildTestPod("spread", 300, 64 << 20, WithNamespace("ns1"), WithLabels({"app": "spread"}))
    spread.topology_spread = [TopologySpreadConstraint(1, LABEL_HOSTNAME, LabelSelector(match_labels={"app": "spread"}))]
    groups = [PodEquivalenceGroup([p.clone() for _ in range(n)]) for p, n in ((plain, 6), (port, 2), (shy, 2), (spread, 4))]
    for g in groups:
        for i, p in enumerate(g.pods):
            p.name = "%s-%d" % (p.name, i)
    return full, templates, groups


def test_filter_pass_places_pods_on_upcoming_copies(engines, oracle):
    """Pods that fit only a new node: before the copies the estimate asks for nodes of t0; with the copies the filter pass
    places them there, and after cae_force_add_pods the estimate no longer asks for them.  Every step against a fresh
    load of the stated objects and the oracle."""
    eng, fresh = engines(True)
    cluster, templates, groups = _provisioned_world()
    enc, enc0 = _encoder(cluster, templates, groups)
    eng.load(enc0)
    caps = np.full(enc0.T, 100, np.int32)
    nc0 = eng.estimate_all(caps)[0].copy()
    assert nc0[0] >= 2
    copies = upcoming_node_infos([int(nc0[0]), 2, 2], templates)     # t2 twice: two copies at their pod limit
    up = enc.upcoming_nodes(copies, cluster)
    assert eng.add_upcoming_nodes(up)
    after = enc0.apply_upcoming(up)
    _check(eng, fresh, oracle, after, True)
    N = after.struct.num_cluster_nodes
    order = np.arange(after.P, dtype=np.int32)
    assigned, _, _ = eng.filter_schedulable(order)
    want = oracle.filter_schedulable(after, order)[0]
    assert np.array_equal(assigned[:after.P], want[:after.P])
    placed = np.flatnonzero(assigned[:after.P] >= 0)
    assert len(placed) and (assigned[placed] >= 2).all() and (assigned[placed] < N).all()
    # the DaemonSet host port and the anti-affinity to the DaemonSet pods keep those pods off t1's copies
    t1_rows = [2 + j for j, (t, _) in enumerate(copies) if t == 1]
    g_off = after.arrays["group_off"]
    for g in (1, 2):
        assert not np.isin(assigned[g_off[g]:g_off[g + 1]], t1_rows).any()
    # t2's copies are at their pod limit: nothing lands there
    t2_rows = [2 + j for j, (t, _) in enumerate(copies) if t == 2]
    assert not np.isin(assigned[placed], t2_rows).any()
    moved, cur = assigned[placed], after.apply_force_add(placed, assigned[placed])[0]
    eng.force_add_pods(placed, moved)
    _check(eng, fresh, oracle, cur, True)
    nc1 = eng.estimate_all(caps)[0]
    fresh.load(cur)
    assert np.array_equal(nc1, fresh.estimate_all(caps)[0])
    assert nc1[0] < nc0[0]


def test_next_loop_replaces_copies_with_the_registered_node(engines, oracle):
    """loop 1: copies added; loop 2, in one call: last loop's copies removed, one registered node arrives as a churn-added
    row, a new copy is added"""
    eng, fresh = engines(False)
    cluster, templates, groups = _provisioned_world()
    enc, enc0 = _encoder(cluster, templates, groups)
    eng.load(enc0)
    up = enc.upcoming_nodes(upcoming_node_infos([2, 1, 0], templates), cluster)
    assert eng.add_upcoming_nodes(up)
    cur = enc0.apply_upcoming(up)
    _check(eng, fresh, oracle, cur, False)
    real = sanitized_node_info(templates[0], "real")
    up2 = enc.upcoming_nodes(upcoming_node_infos([1, 0, 1], templates), cluster + [real])
    assert up2.churn.num_removed == 3 and up2.churn.num_added == 1 and up2.num_upcoming == 2
    assert eng.add_upcoming_nodes(up2)
    cur = cur.apply_upcoming(up2)
    _check(eng, fresh, oracle, cur, False)


@pytest.mark.parametrize("shape", ["c3", "c4"])
def test_ten_chained_loops(engines, oracle, shape):
    """upcoming calls (with churns that remove the previous copies) interleaved with cae_load_pending, cae_load_nodes,
    cae_load_pods, cae_load_templates and cae_force_add_pods, in both orders"""
    eng, fresh = engines(True)
    cur = _gen(shape)
    eng.load(cur)
    prev = []
    for k in range(10):
        churn, pending = synth.node_scale(cur, 500 + k, 1 + k % 3, k % 3, k)
        churn = churn.replace(removed=sorted(set(churn.arrays["removed"].tolist()) | set(prev) - set(churn.changed.arrays["row"].tolist())))
        tmpl = [(3 * k + j) % cur.T for j in range(1 + k % 4)]
        up = _copies(cur, tmpl, churn, (0,) if k % 3 == 0 else ())
        if k % 2:
            assert eng.load_pending(pending) and eng.add_upcoming_nodes(up)
        else:
            assert eng.add_upcoming_nodes(up) and eng.load_pending(pending)
        cur = pending.apply_upcoming(up)
        n_new = cur.struct.num_cluster_nodes
        prev = list(range(n_new - len(tmpl), n_new))
        delta, pending = synth.node_churn(cur, 700 + k, 2 + k)
        if k % 2:
            assert eng.load_nodes(delta) and eng.load_pending(pending)
        else:
            assert eng.load_pending(pending) and eng.load_nodes(delta)
        cur = pending.apply_node_delta(delta)
        if k % 5 == 2:   # new workloads arrive, some finish
            pd = synth.pod_churn(cur, 900 + k, 2, 1)
            nxt = cur.apply_pod_delta(pd)
            assert eng.load_pods(pd, nxt) == 0
            cur = nxt
        if k % 5 == 3:   # node-group templates change, one goes away, one is added
            td = synth.template_churn(cur, 950 + k, 2, 1, 1)
            nxt = cur.apply_template_delta(td)
            assert eng.load_templates(td, nxt)
            cur = nxt
        if k % 3 == 1:   # the filter pass's placements force-added
            order = np.arange(min(cur.P, 300), dtype=np.int32)
            eng.enc = cur
            assigned = eng.filter_schedulable(order)[0][:cur.P]
            pods = np.flatnonzero(assigned >= 0).astype(np.int32)
            if len(pods):
                nxt = cur.apply_force_add(pods, assigned[pods])[0]
                assert eng.force_add_pods(pods, assigned[pods]) is not False
                cur = nxt
        _check(eng, fresh, oracle, cur, True, with_oracle=k in (4, 9))


def test_empty_and_template_free_calls(engines, oracle):
    from kubernetes_autoscaler_b200.engine import EngineError
    eng, fresh = engines(False)
    enc = _gen("c3")
    eng.load(enc)
    before = _results(eng, enc)
    assert eng.add_upcoming_nodes(UpcomingNodes())
    assert eng.stats().h2d_bytes == 0
    _assert_same(_results(eng, enc), before, "empty call")
    # T = 0: there is no template to copy
    t0 = _gen("c4", templates=0, pods=600)
    eng.load(t0)
    before = _results(eng, t0)
    with pytest.raises(EngineError, match="status -2"):
        eng.add_upcoming_nodes(UpcomingNodes(template_idx=[0], name=[5000], labelset=[0]))
    _assert_same(_results(eng, t0), before, "T = 0")
    # T = 0 with a churn only: the churn applies
    churn, pending = synth.node_scale(t0, 9, 2, 3)
    up = UpcomingNodes(churn)
    assert eng.add_upcoming_nodes(up)
    _check(eng, fresh, oracle, pending.apply_upcoming(up), False)


def test_refusals_leave_the_engine_unchanged(engines):
    from kubernetes_autoscaler_b200.engine import EngineError
    eng, _ = engines(False)
    enc = _gen("c3")
    N, T = enc.struct.num_cluster_nodes, enc.T
    eng.load(enc)
    before = _results(eng, enc)
    ok = _copies(enc, [0, 1, 2], synth.node_scale(enc, 4, 3, 3, 4)[0])
    # status 2: the rows, the copies counted (no copy array is read) ...
    huge_rows = ok.replace()
    huge_rows.struct.num_upcoming = 2 ** 31 - 1 - N - 2 * T + 1
    # ... and the resident pods, the copies' template pods counted: one added row whose offsets (never its pod-spec ids)
    # leave room for every pod but the copies' last one
    total = int(enc.arrays["node_pod_off"][-1])
    tp = int(np.diff(enc.arrays["node_pod_off"])[N:N + 3].sum())
    assert tp > 0
    big = NodeChurn(name=[9000], labelset=[0], taint_list=[0], unschedulable=[0], allowed_pods=[10],
                    pod_off=np.array([0, 2 ** 31 - 1 - total - tp + 1], np.int32), pod_spec=[0])
    huge_pods = _copies(enc, [0, 1, 2], big)
    refused = {"node rows": huge_rows, "resident pods": huge_pods}
    for what, u in refused.items():
        assert not eng.add_upcoming_nodes(u), what
        _assert_same(_results(eng, enc), before, "after a refused call (%s)" % what)
    # status -2
    nl = enc.struct.num_labelsets + ok.churn.changed.struct.num_new_labelsets
    bad = {
        "template index negative": ok.replace(template_idx=[0, -1, 2]),
        "template index past T": ok.replace(template_idx=[0, T, 2]),
        "name negative": ok.replace(name=[5000, -1, 5002]),
        "label set past the tails": ok.replace(labelset=[0, nl, 0]),
        "label set negative": ok.replace(labelset=[0, -1, 0]),
        "churn malformed": ok.replace(churn=ok.churn.replace(removed=[N])),
    }
    for field in ("template_idx", "name", "labelset"):
        u = ok.replace()
        setattr(u.struct, field, None)
        bad["null " + field] = u
    u = ok.replace()
    u.struct.abi_version = 99
    bad["abi version"] = u
    u = ok.replace(churn=ok.churn.replace())
    u.churn.struct.abi_version = 99
    bad["abi version of the churn"] = u
    u = ok.replace()
    u.struct.num_upcoming = -1
    bad["negative count"] = u
    for what, u in bad.items():
        with pytest.raises(EngineError, match="status -2"):
            eng.add_upcoming_nodes(u)
        assert eng.add_upcoming_nodes(UpcomingNodes()), what
    _assert_same(_results(eng, enc), before, "after malformed calls")


def _rank_answers(e, enc):
    from delta_harness import _filter_args
    e.enc = enc
    bits, reasons, count = e.feasibility()
    out = {"bits": bits.copy(), "reasons": reasons.copy(), "count": count.copy(), "groups": e.feasibility_groups()}
    for cap in (40, 0):
        out["est%d" % cap] = tuple(x.copy() for x in e.estimate_all(np.full(enc.T, cap, np.int32)))
        out["waste%d" % cap] = e.waste_scores()
    out["filter"] = e.filter_schedulable(*_filter_args(enc))
    return out


@pytest.mark.parametrize("W", [2, 3, 8])
def test_every_rank_applies_the_same_call(oracle, W):
    """At world_size W every rank applies the same call (copies with a churn): each rank's answers equal those of the same
    rank freshly loaded with the objects after the call, and rank 0's dense rows equal the oracle's"""
    import __graft_entry__ as g
    from delta_harness import _equal
    from kubernetes_autoscaler_b200.engine import Engine, shard_pods, unpack_bits
    g.build()
    enc = _gen("c3", pods=1000, templates=24, cluster_nodes=40)
    churn, pending = synth.node_scale(enc, 61, 3, 2, 4)
    up = _copies(enc, [0, 5, 5, 23], churn, (1,))
    after = pending.apply_upcoming(up)
    for rank in range(W):
        e, twin = Engine(device=0, rank=rank, world_size=W, want_reasons=True), Engine(device=0, rank=rank, world_size=W, want_reasons=True)
        try:
            e.load(enc)
            assert e.add_upcoming_nodes(up) and e.load_pending(pending)
            got = _rank_answers(e, after)
            twin.load(after)
            want = _rank_answers(twin, after)
            for k in want:
                assert _equal(got[k], want[k]), "W=%d rank %d: %s differs from a fresh load" % (W, rank, k)
            if rank == 0:
                pb, pe = shard_pods(after.P, 0, W)
                reasons = oracle.feasibility_dense(after, p_range=(pb, pe))[0]
                assert np.array_equal(got["reasons"], reasons)
                assert np.array_equal(unpack_bits(got["bits"], pe - pb), reasons == 0)
        finally:
            e.close()
            twin.close()


def test_whole_snapshot_calls_after_the_copies(engines, oracle):
    """group reasons, similar node groups, scale-down eligibility, the filter pass, the removal batch (persisted or not)
    and the capacity batch after the call equal a fresh load's; so does a removal batch whose candidates and destinations
    leave the copies out, as the planner's are"""
    from test_gpu_shards import _whole_answers
    from delta_harness import _equal
    eng, fresh = engines(True)
    enc = _gen("c4")
    churn, pending = synth.node_scale(enc, 71, 3, 4, 6)
    up = _copies(enc, [2, 2, 7, 11, 0], churn, (3,))
    after = pending.apply_upcoming(up)
    eng.load(enc)
    assert eng.add_upcoming_nodes(up) and eng.load_pending(pending)
    fresh.load(after)
    for e in (eng, fresh):
        e.enc = after
    N, P = after.struct.num_cluster_nodes, after.P
    real = N - 5                                          # the copies are the last five cluster rows
    dest = (np.arange(N) < real).astype(np.uint8)
    cand = np.array([0, 4, real - 1], np.int32)
    move_off = np.array([0, 3, 7, 12], np.int32)
    move_pod = (np.arange(12) * 41 % P).astype(np.int32)
    got = [e.simulate_removals(cand, move_off, move_pod, dest, None, last_index=0) for e in (eng, fresh)]
    assert _equal(got[0], got[1]), "removal batch with the copies left out"
    S = after.struct.num_podspecs
    ds = np.arange(0, S, max(1, S // 12), dtype=np.int32)[:12]
    got = [tuple(x.copy() for x in e.template_daemonsets(ds)) for e in (eng, fresh)]
    assert _equal(got[0], got[1]), "template DaemonSet verdicts"
    want = _whole_answers(fresh, after)
    have = _whole_answers(eng, after)
    for k in want:
        assert _equal(have[k], want[k]), "%s differs from a fresh load" % k
    assert np.array_equal(have["groups"], oracle.feasibility_groups(after))
    # the resident removals of real candidates, their pods moving to real rows only (after the persisted batch above, so
    # both engines start from the same persisted state)
    off = after.arrays["node_pod_off"]
    rcand = np.array([1, 6, real - 2], np.int32)
    cnt = [min(3, int(off[c + 1] - off[c])) for c in rcand]
    move_off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    move_slot = np.concatenate([np.arange(n) for n in cnt]).astype(np.int32)
    got = [e.simulate_resident_removals(rcand, move_off, move_slot, dest) for e in (eng, fresh)]
    assert _equal(tuple(np.asarray(x).copy() for x in got[0]), tuple(np.asarray(x).copy() for x in got[1])), "resident removals"
