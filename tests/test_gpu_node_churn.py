"""cae_load_node_churn on the GPU: after cluster nodes are removed and added (with or without dirty rows) every entry point
answers bit-identically to a second engine freshly loaded with EncodedObjects.apply_node_churn(...), and to the oracle
where that is affordable — dense bits / reasons / counts, group reasons, Estimate() (capped, unlimited, RAW lastIndex),
waste and price scores, the filter-out-schedulable pass, the scale-down batch.  Chained churns interleaved with
cae_load_nodes and cae_load_pending, boundary churns, and every refusal (status 2) and malformed input (status -2) with the
engine left as it was."""
import copy

import numpy as np
import pytest

from delta_harness import SHAPES, _assert_same, _check, _equal, _filter_args, _gen, _results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import Encoder, NodeChurn, NodeDelta
from kubernetes_autoscaler_b200.objects import BuildTestPod, LabelSelector, NodeInfo, PodAffinityTerm, WithLabels, WithNamespace, \
    WithPodAntiAffinity

pytestmark = pytest.mark.gpu

KINDS = {"removes": (5, 0, 0), "adds": (0, 6, 0), "both": (4, 7, 0), "both+dirty": (6, 5, 9)}


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_churn_matches_full_load(engines, oracle, shape, want_reasons):
    eng, fresh = engines(want_reasons)
    enc = _gen(shape)
    for k, (kind, (nr, na, nd)) in enumerate(sorted(KINDS.items())):
        churn, pending = synth.node_scale(enc, 11 + k, nr, na, nd)
        assert churn.num_removed == nr and churn.num_added == na
        after = pending.apply_node_churn(churn)
        eng.load(enc)
        assert eng.load_node_churn(churn), kind
        if nd:
            assert eng.load_pending(pending)
        _check(eng, fresh, oracle, after, want_reasons, with_oracle=want_reasons)
    # the reverse order: pending rows first, then the nodes
    eng.load(enc)
    assert eng.load_pending(pending) and eng.load_node_churn(churn)
    _check(eng, fresh, oracle, after, want_reasons, with_oracle=False)


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_ten_chained_churns(engines, oracle, shape):
    """churns interleaved with cae_load_nodes and cae_load_pending, in both orders"""
    eng, fresh = engines(True)
    cur = _gen(shape)
    eng.load(cur)
    for k in range(10):
        churn, pending = synth.node_scale(cur, 200 + k, 1 + k % 4, 1 + (k * 3) % 5, 2 * k)
        if k % 2:
            assert eng.load_pending(pending) and eng.load_node_churn(churn)
        else:
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
        cur = pending.apply_node_churn(churn)
        delta, pending = synth.node_churn(cur, 300 + k, 3 + k)
        if k % 2:
            assert eng.load_nodes(delta) and eng.load_pending(pending)
        else:
            assert eng.load_pending(pending) and eng.load_nodes(delta)
        cur = pending.apply_node_delta(delta)
        _check(eng, fresh, oracle, cur, True, with_oracle=k in (4, 9))


def _labels(enc, ls):
    a = enc.arrays
    return dict(zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist(), a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist()))


def _row_churn(enc, removed=(), copies=(), dirty=(), new_values=0):
    """A churn built from existing rows: `copies` = [(row, label changes)] added nodes shaped like `row` with a new name,
    `dirty` = [(row, label changes)]; a label change to value "new" takes the next new value id."""
    a, s = enc.arrays, enc.struct
    off = a["node_pod_off"]
    names_next = int(a["node_name"].max()) + 1
    vals = [s.num_values]
    pairs, ls_off = [], [0]

    def relabel(row, change):
        lab = _labels(enc, int(a["node_labelset"][row]))
        for k, v in change.items():
            if v is None:
                lab.pop(k, None)
            elif v == "new":
                lab[k] = vals[0]
                vals[0] += 1
            else:
                lab[k] = v
        pairs.append(sorted(lab.items()))
        ls_off.append(ls_off[-1] + len(pairs[-1]))
        return s.num_labelsets + len(pairs) - 1

    d_rows = [r for r, _ in dirty]
    d_ls = [relabel(r, ch) for r, ch in dirty]
    c_ls = [relabel(r, ch) for r, ch in copies]
    nv = vals[0] - s.num_values
    lists = [a["node_pod_spec"][off[r]:off[r + 1]] for r in d_rows]
    d_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
    changed = NodeDelta(value_is_int=np.zeros(nv), value_int=np.zeros(nv), ls_off=ls_off,
                        ls_key=[k for p in pairs for k, _ in p], ls_val=[v for p in pairs for _, v in p],
                        row=d_rows, labelset=d_ls, taint_list=a["node_taint_list"][d_rows],
                        unschedulable=a["node_unschedulable"][d_rows], alloc=a["node_alloc"][d_rows],
                        allowed_pods=a["node_allowed_pods"][d_rows], pod_off=d_off,
                        pod_spec=np.concatenate(lists) if lists else [])
    rows = [r for r, _ in copies]
    lists = [a["node_pod_spec"][off[r]:off[r + 1]] for r in rows]
    return NodeChurn(changed, removed=sorted(removed), name=[names_next + i for i in range(len(rows))], labelset=c_ls,
                     taint_list=a["node_taint_list"][rows], unschedulable=a["node_unschedulable"][rows], alloc=a["node_alloc"][rows],
                     allowed_pods=a["node_allowed_pods"][rows], pod_off=np.concatenate([[0], np.cumsum([len(x) for x in lists])]),
                     pod_spec=np.concatenate(lists) if lists else [])


def _zone_of(enc, row):
    return _labels(enc, int(enc.arrays["node_labelset"][row])).get(synth.K_ZONE)


def test_boundary_churns(engines, oracle):
    eng, fresh = engines(False)
    enc = _gen("c3")
    N = enc.struct.num_cluster_nodes
    # an empty call: a no-op that uploads nothing
    eng.load(enc)
    before = _results(eng, enc)
    assert eng.load_node_churn(NodeChurn())
    assert eng.stats().h2d_bytes == 0
    _assert_same(_results(eng, enc), before, "empty churn")
    # every cluster node removed (N' = 0), then nodes added to the empty cluster
    eng.load(enc)
    gone = NodeChurn(removed=np.arange(N))
    assert eng.load_node_churn(gone)
    cur = enc.apply_node_churn(gone)
    assert cur.struct.num_cluster_nodes == 0
    _check(eng, fresh, oracle, cur, False)
    back = _row_churn(enc, copies=[(r, {synth.K_HOST: "new"}) for r in (0, 5, 9)])
    assert eng.load_node_churn(back)
    cur = cur.apply_node_churn(back)
    _check(eng, fresh, oracle, cur, False)
    # nodes added to a load with N = 0
    empty = _gen("c3", cluster_nodes=0)
    eng.load(empty)
    churn, pending = synth.node_scale(empty, 3, 0, 9)
    assert churn.num_added == 9
    assert eng.load_node_churn(churn)
    _check(eng, fresh, oracle, pending.apply_node_churn(churn), False)
    # the first and the last row removed
    eng.load(enc)
    ends = NodeChurn(removed=[0, N - 1])
    assert eng.load_node_churn(ends)
    _check(eng, fresh, oracle, enc.apply_node_churn(ends), False)
    # a node removed and one with the same name added: it becomes the last row
    eng.load(enc)
    same = _row_churn(enc, removed=[7], copies=[(7, {})])
    same.arrays["name"][:] = enc.arrays["node_name"][7]
    same = same.replace()
    assert eng.load_node_churn(same)
    cur = enc.apply_node_churn(same)
    assert cur.arrays["node_name"][N - 1] == enc.arrays["node_name"][7]
    _check(eng, fresh, oracle, cur, False)
    # a new zone value: a domain appears
    eng.load(enc)
    nz = _row_churn(enc, copies=[(3, {synth.K_HOST: "new", synth.K_ZONE: "new"}), (4, {synth.K_HOST: "new"})])
    assert eng.load_node_churn(nz)
    cur = enc.apply_node_churn(nz)
    zones = {_zone_of(cur, r) for r in range(cur.struct.num_cluster_nodes)}
    assert len(zones) == len({_zone_of(enc, r) for r in range(N)}) + 1
    _check(eng, fresh, oracle, cur, False)
    # the last node of a zone removed, with minDomains in play (C3 spreads on zone with minDomains 1 or 3)
    zone_rows = {}
    for r in range(N):
        zone_rows.setdefault(_zone_of(enc, r), []).append(r)
    smallest = min(zone_rows.values(), key=len)
    eng.load(enc)
    lz = NodeChurn(removed=smallest)
    assert eng.load_node_churn(lz)
    cur = enc.apply_node_churn(lz)
    assert len({_zone_of(cur, r) for r in range(cur.struct.num_cluster_nodes)}) == len(zone_rows) - 1
    assert any(v > 1 for v in enc.arrays["pts_min_domains"])
    _check(eng, fresh, oracle, cur, False)
    # a dirty row moving zone: a churn rebuilds the domains, cae_load_nodes refuses the same delta
    other = next(z for z in zone_rows if z != _zone_of(enc, 2))
    mz = _row_churn(enc, dirty=[(2, {synth.K_ZONE: other})])
    eng.load(enc)
    assert not eng.load_nodes(mz.changed)
    assert eng.load_node_churn(mz)
    _check(eng, fresh, oracle, enc.apply_node_churn(mz), False)


def test_scale_down_batch_after_churn(engines):
    """a T = 0 load (what the scale-down batch uses), a churn, then cae_simulate_removals and the filter pass with a non-zero
    lastIndex, against a fresh load"""
    eng, fresh = engines(False)
    enc = _gen("c4", templates=0, pods=600)
    assert enc.T == 0
    churn, pending = synth.node_scale(enc, 5, 6, 4, 5)
    after = pending.apply_node_churn(churn)
    eng.load(enc)
    assert eng.load_node_churn(churn) and eng.load_pending(pending)
    fresh.load(after)
    N, P = after.struct.num_cluster_nodes, after.P
    cand = np.array([0, 3, N - 1, 7, N - 2, 3], np.int32)       # row 3 twice: its pods are listed again
    move_off = np.array([0, 4, 9, 9, 15, 20, 24], np.int32)
    move_pod = np.concatenate([np.arange(20), np.arange(4, 8)]).astype(np.int32)
    dest = (np.arange(N) % 5 != 1).astype(np.uint8)
    hint = np.where(np.arange(P) % 9 == 0, np.arange(P) % max(N, 1), -1).astype(np.int32)
    for persist in (False, True):
        for li in (0, 3, 5 * N + 2):
            eng.enc = fresh.enc = after
            got = eng.simulate_removals(cand, move_off, move_pod, dest, hint, last_index=li, persist=persist)
            want = fresh.simulate_removals(cand, move_off, move_pod, dest, hint, last_index=li, persist=persist)
            assert all(_equal(x, y) for x, y in zip(got, want)), (persist, li)
    for li in (1, N + 4):
        assert _equal(eng.filter_schedulable(*_filter_args(after, last=li)), fresh.filter_schedulable(*_filter_args(after, last=li)))


def _anti_world():
    """An Encoder whose spec table holds an anti-affinity spec no pod uses at load time."""
    from test_node_delta_host import _world
    cluster, templates, groups = _world()
    enc = Encoder()
    for ni in cluster:
        enc.add_cluster_node(ni)
    for ni in templates:
        enc.add_template(ni)
    for g in groups:
        enc.add_group(g)
    lonely = BuildTestPod("lonely", 100, 100, WithNamespace("ns1"), WithLabels({"app": "lonely"}),
                          WithPodAntiAffinity(PodAffinityTerm(LabelSelector(match_labels={"app": "lonely"}), "pool")))
    enc.podspec(lonely)
    return enc, enc.finish(), cluster, lonely


def test_refusals_leave_the_engine_unchanged(engines):
    eng, _ = engines(False)
    enc = _gen("c3")
    N = enc.struct.num_cluster_nodes
    eng.load(enc)
    before = _results(eng, enc)
    ok = synth.node_scale(enc, 4, 3, 3, 4)[0]
    huge_rows = ok.replace()
    huge_rows.struct.num_added = 2 ** 31 - 1 - N - 2 * enc.T + 4   # N' + 2T > 2^31 - 1; no added array is read
    huge_dict = ok.replace(changed=ok.changed.replace())
    huge_dict.changed.struct.num_new_values = 2 ** 31 - enc.struct.num_values
    refused = {
        "node rows": huge_rows,
        "resident pods": ok.replace(pod_off=np.array([0, 1, 2, 2 ** 31 - 64], np.int32), pod_spec=[0] * 3),
        "dictionary": huge_dict,
    }
    for what, c in refused.items():
        assert not eng.load_node_churn(c), what
        _assert_same(_results(eng, enc), before, "after a refused churn (%s)" % what)
    # a resident pod (of an added or a dirty row) whose anti-affinity spec was in no pod of the last load
    for dirty in (False, True):
        enc_w, enc2, cluster, lonely = _anti_world()
        eng.load(enc2)
        before2 = _results(eng, enc2)
        new = cluster[:2] + cluster[3:]
        if dirty:
            new[1].pods.append(lonely)
        else:
            extra = NodeInfo(copy.deepcopy(cluster[0].node), [lonely])
            extra.node.name = "extra"
            new.append(extra)
        c = enc_w.node_churn(new)
        assert not eng.load_node_churn(c)
        _assert_same(_results(eng, enc2), before2, "after a refused anti-affinity resident")


def test_malformed_churns(engines):
    from kubernetes_autoscaler_b200.engine import EngineError
    eng, _ = engines(False)
    enc = _gen("c2")
    N, S = enc.struct.num_cluster_nodes, enc.struct.num_podspecs
    eng.load(enc)
    before = _results(eng, enc)
    ok = synth.node_scale(enc, 4, 3, 3, 4)[0]
    rows = ok.changed.arrays["row"]
    nl = enc.struct.num_labelsets + ok.changed.struct.num_new_labelsets
    nt = enc.struct.num_taint_lists + ok.changed.struct.num_new_taint_lists
    clean = [r for r in range(N) if r not in set(rows.tolist())]
    bad = {
        "dirty row out of range": ok.replace(changed=ok.changed.replace(row=np.concatenate([rows[:-1], [N]]))),
        "removed out of range": ok.replace(removed=[clean[0], N]),
        "removed negative": ok.replace(removed=[-1, clean[0]]),
        "removed not increasing": ok.replace(removed=[clean[1], clean[0]]),
        "removed twice": ok.replace(removed=[clean[0], clean[0]]),
        "removed and dirty": ok.replace(removed=sorted([clean[0], int(rows[0])])),
        "added label set": ok.replace(labelset=np.full(3, nl, np.int32)),
        "added taint list": ok.replace(taint_list=np.full(3, nt, np.int32)),
        "added name": ok.replace(name=[-1, 5000, 5001]),
        "added pod spec": ok.replace(pod_spec=np.full(len(ok.arrays["pod_spec"]), S, np.int32)),
        "added offsets start": ok.replace(pod_off=ok.arrays["pod_off"] + 1),
        "added offsets decrease": ok.replace(pod_off=np.array([0, 5, 3, len(ok.arrays["pod_spec"])], np.int32)),
    }
    for field in ("name", "labelset", "taint_list", "unschedulable", "alloc", "allowed_pods", "pod_off"):
        c = ok.replace()
        setattr(c.struct, field, None)
        bad["null " + field] = c
    c = ok.replace()
    c.struct.removed = None
    bad["null removed"] = c
    c = ok.replace()
    c.struct.abi_version = 99
    bad["abi version"] = c
    c = ok.replace(changed=ok.changed.replace())
    c.changed.struct.abi_version = 99
    bad["abi version of changed"] = c
    c = ok.replace()
    c.struct.num_added = -1
    bad["negative count"] = c
    for what, c in bad.items():
        with pytest.raises(EngineError, match="status -2"):
            eng.load_node_churn(c)
        assert eng.load_node_churn(NodeChurn()), what
    _assert_same(_results(eng, enc), before, "after malformed churns")
