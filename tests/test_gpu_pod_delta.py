"""cae_load_pods on the GPU: after new pod specs arrive and the pending list is replaced, every entry point answers
bit-identically to a second engine freshly loaded with EncodedObjects.apply_pod_delta(...), and to the oracle where that
is affordable (the results of tests/delta_harness.py: dense bits / reasons / counts, group reasons, Estimate()
capped and unlimited, RAW lastIndex, waste and price scores, the filter pass).  Chained deltas interleaved with
cae_load_pending, cae_load_nodes and cae_load_node_churn (node calls naming the new specs as residents), boundaries, and
refusals / malformed input with the engine left as it was."""
import numpy as np
import pytest

from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import PodDelta

from delta_harness import SHAPES, _assert_same, _check, _gen, _results, engines  # noqa: F401  (engines: fixture)
from test_node_delta_host import _encoder, _world
from test_pod_delta_host import new_workloads
from test_node_churn_host import _new_node

pytestmark = pytest.mark.gpu

_SPEC_COLS = ("ps_namespace", "ps_labelset", "ps_tol_list", "ps_naff", "ps_node_name", "ps_port_list", "ps_pts_list",
              "ps_aff_list", "ps_anti_list", "ps_terminating", "ps_hostname_spread")


def _synth_delta(enc, seed, new_specs, keep=0.75, grow=1):
    """New specs copied from resident ones with new cpu requests (new rank values), and a regrouped pending list: a
    shuffled subset of the old groups (each repeated `grow` times) plus one group per new spec."""
    a, S = enc.arrays, enc.struct.num_podspecs
    rng = np.random.default_rng(seed)
    src = rng.integers(0, S, new_specs)
    cols = {nm: a[nm][src] for nm in _SPEC_COLS}
    req = a["ps_req"][src].copy()
    req[:, 0] = req[:, 0] + 7 * (np.arange(new_specs) + 1)
    go = a["group_off"]
    E = len(go) - 1
    old = [a["pend_spec"][go[g]:go[g + 1]] for g in rng.permutation(E)[:int(E * keep)]] * grow
    pend = old + [np.full(1 + i % 5, S + i, np.int32) for i in range(new_specs)]
    off = np.concatenate([[0], np.cumsum([len(p) for p in pend])]).astype(np.int32)
    return PodDelta(ps_req=req, group_off=off, pend_spec=np.concatenate(pend) if pend else [], **cols)


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
def test_object_world_deltas(engines, oracle, want_reasons):
    """new workloads with new labels, namespaces, a new topology key, a first anti-affinity spec and host ports; then a
    second delta whose new spec is bound to a node by the node delta that follows"""
    eng, fresh = engines(want_reasons)
    cluster, templates, groups = _world()
    enc, cur = _encoder(cluster, templates, groups)
    eng.load(cur)
    new = groups[2:3] + new_workloads()
    delta = enc.pod_delta(new)
    cur = cur.apply_pod_delta(delta)
    assert eng.load_pods(delta, cur) == 0
    _check(eng, fresh, oracle, cur, want_reasons)
    newer = new_workloads()[1:] + groups[:1]
    bound = newer[0].pods[0].clone()
    bound.node_name = cluster[1].node.name
    cluster[1].pods.append(bound)
    d2 = enc.pod_delta(newer, residents=[cluster[1]])
    nd = enc.node_delta([(1, cluster[1])])
    cur = cur.apply_pod_delta(d2)
    assert eng.load_pods(d2, cur) == 0 and eng.load_nodes(nd)
    cur = cur.apply_node_delta(nd)
    _check(eng, fresh, oracle, cur, want_reasons)
    joined = _new_node("n9", "z0", [newer[2].pods[0]])
    d3 = enc.pod_delta(newer, residents=[joined])
    churn = enc.node_churn(cluster + [joined])
    cur = cur.apply_pod_delta(d3)
    assert eng.load_pods(d3, cur) == 0 and eng.load_node_churn(churn)
    cur = cur.apply_node_churn(churn)
    _check(eng, fresh, oracle, cur, want_reasons)


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_synth_deltas_match_full_load(engines, oracle, shape):
    """regrouping under counters (which cae_load_pending refuses), P and E past the load's buffers, P = 0"""
    eng, fresh = engines(True)
    enc = _gen(shape)
    for k, (n_new, keep, grow) in enumerate(((5, 0.75, 1), (12, 1.0, 3), (0, 0.0, 1), (3, 0.5, 1))):
        eng.load(enc)
        delta = _synth_delta(enc, 40 + k, n_new, keep, grow)
        after = enc.apply_pod_delta(delta)
        assert eng.load_pods(delta, after) == 0
        _check(eng, fresh, oracle, after, True, with_oracle=k == 0)


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_ten_chained_deltas(engines, oracle, shape):
    """pod deltas interleaved with cae_load_pending, cae_load_nodes and cae_load_node_churn, whose rows name the new
    specs as residents"""
    eng, fresh = engines(True)
    cur = _gen(shape)
    eng.load(cur)
    for k in range(10):
        delta = _synth_delta(cur, 500 + k, 1 + k % 4, keep=0.6 + 0.04 * k)
        cur = cur.apply_pod_delta(delta)
        assert eng.load_pods(delta, cur) == 0
        if k % 3 == 0:
            nd, pending = synth.node_churn(cur, 600 + k, 2 + k)
            S = cur.struct.num_podspecs
            spec = nd.arrays["pod_spec"].copy()
            spec[::3] = S - 1                                    # the newest spec becomes resident
            nd = nd.replace(pod_spec=spec)
            assert eng.load_nodes(nd) and eng.load_pending(pending)
            cur = pending.apply_node_delta(nd)
        elif k % 3 == 1:
            churn, pending = synth.node_scale(cur, 700 + k, 1 + k % 3, 2, 1)
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
            cur = pending.apply_node_churn(churn)
        _check(eng, fresh, oracle, cur, True, with_oracle=k in (4, 9))


def test_refusals_leave_the_engine_unchanged(engines):
    eng, fresh = engines(False)
    enc = _gen("c3")
    eng.load(enc)
    want = _results(eng, enc)
    S, NPL = enc.struct.num_podspecs, enc.struct.num_port_lists
    ok = _synth_delta(enc, 9, 3)
    bad = [ok.replace(pend_spec=np.where(np.arange(len(ok.arrays["pend_spec"])) == 0, S + 3, ok.arrays["pend_spec"])),
           ok.replace(group_off=ok.arrays["group_off"][:-1]),
           ok.replace(ps_labelset=np.full(3, 1 << 30)),
           ok.replace(ls_off=[1, 2], ls_key=[3], ls_val=[0]),
           ok.replace(ls_off=[0, 2], ls_key=[5, 3], ls_val=[0, 0]),
           ok.replace(req_key=[1], req_op=[9], req_val_off=[0, 0]),
           ok.replace(ps_req=np.full((3, 8), -5))]
    for d in bad:
        with pytest.raises(RuntimeError):
            eng.load_pods(d)
    # status 1: more than 64 host-port sets among pending pods
    n = 70
    ports = PodDelta(port_off=np.arange(n + 1), port_ip=np.zeros(n), port_proto=np.zeros(n), port_num=9000 + np.arange(n),
                     **{nm: np.repeat(enc.arrays[nm][:1], n) for nm in _SPEC_COLS if nm != "ps_port_list"},
                     ps_port_list=NPL + np.arange(n), ps_req=np.repeat(enc.arrays["ps_req"][:1], n, axis=0),
                     group_off=np.arange(n + 1), pend_spec=S + np.arange(n))
    assert eng.load_pods(ports) == 1
    _assert_same(_results(eng, enc), want, "after refusals")
    # the engine still takes a good delta, and cae_load_pending judges against it
    after = enc.apply_pod_delta(ok)
    assert eng.load_pods(ok, after) == 0
    assert eng.load_pending(after)
    fresh.load(after)
    _assert_same(_results(eng, after), _results(fresh, after), "after a good delta")


def _new_specs(enc, n, **cols):
    """n new specs shaped like spec 0 (columns overridable), and a pending list of one group per new spec"""
    S = enc.struct.num_podspecs
    base = {nm: np.repeat(enc.arrays[nm][:1], n) for nm in _SPEC_COLS}
    base["ps_req"] = np.repeat(enc.arrays["ps_req"][:1], n, axis=0)
    base.update(cols)
    return dict(base, group_off=np.arange(n + 1), pend_spec=S + np.arange(n))


def test_c1_shape_and_boundaries(engines, oracle):
    """C1, lut_rows past FEAS_LUT_MAX_ROWS (the bit-sliced dense pass) with the rank field widening, a new active
    resource dim, and the last spec of a topology key leaving"""
    eng, fresh = engines(True)
    enc = synth.generate(1, pods=2000, templates=24, cluster_nodes=32)
    eng.load(enc)
    delta = _synth_delta(enc, 3, 4)
    after = enc.apply_pod_delta(delta)
    assert eng.load_pods(delta, after) == 0
    _check(eng, fresh, oracle, after, True)
    for shape in ("c2", "c3"):
        enc = _gen(shape)
        eng.load(enc)
        n = 1100                                              # 1100 distinct cpu requests: > 1024 threshold rows
        req = np.repeat(enc.arrays["ps_req"][:1], n, axis=0)
        req[:, 0] = 100 + 3 * np.arange(n)
        req[::7, 2] = 1 << 20                                 # ephemeral storage: a dim no pending pod requested
        delta = PodDelta(**_new_specs(enc, n, ps_req=req))
        after = enc.apply_pod_delta(delta)
        assert eng.load_pods(delta, after) == 0
        _check(eng, fresh, oracle, after, True, with_oracle=False)
    # c3 keeps only plain pending specs: every spread key leaves with its last pending spec
    enc = _gen("c3")
    eng.load(enc)
    a = enc.arrays
    plain = [s for s in range(enc.struct.num_podspecs) if a["ps_pts_list"][s] == 0 and a["ps_aff_list"][s] == 0 and a["ps_anti_list"][s] == 0]
    if plain:
        delta = PodDelta(group_off=[0, 3], pend_spec=[plain[0]] * 3)
        after = enc.apply_pod_delta(delta)
        assert eng.load_pods(delta, after) == 0
        _check(eng, fresh, oracle, after, True)


def test_scale_down_batch_after_pod_delta(engines):
    """cae_simulate_removals and the filter pass with non-zero lastIndex after cae_load_pods, against a fresh load"""
    from delta_harness import _equal, _filter_args
    eng, fresh = engines(False)
    enc = _gen("c4", templates=0, pods=600)
    eng.load(enc)
    delta = _synth_delta(enc, 17, 6)
    after = enc.apply_pod_delta(delta)
    assert eng.load_pods(delta, after) == 0
    fresh.load(after)
    N, P = after.struct.num_cluster_nodes, after.P
    cand = np.array([0, 3, N - 1, 7, 3], np.int32)
    move_off = np.array([0, 4, 9, 9, 15, 18], np.int32)
    move_pod = (np.arange(18) % max(P, 1)).astype(np.int32)
    dest = (np.arange(N) % 5 != 1).astype(np.uint8)
    hint = np.where(np.arange(P) % 9 == 0, np.arange(P) % max(N, 1), -1).astype(np.int32)
    for persist in (False, True):
        for li in (0, 5 * N + 2):
            eng.enc = fresh.enc = after
            got = eng.simulate_removals(cand, move_off, move_pod, dest, hint, last_index=li, persist=persist)
            want = fresh.simulate_removals(cand, move_off, move_pod, dest, hint, last_index=li, persist=persist)
            assert all(_equal(x, y) for x, y in zip(got, want)), (persist, li)
    assert _equal(eng.filter_schedulable(*_filter_args(after, last=N + 4)), fresh.filter_schedulable(*_filter_args(after, last=N + 4)))


def test_two_rank_shards():
    """rank 0 and 1 of world 2 on one GPU: each shard's Estimate() after cae_load_pods equals that of a fresh load"""
    from kubernetes_autoscaler_b200.engine import Engine
    enc = _gen("c3")
    delta = _synth_delta(enc, 21, 5)
    after = enc.apply_pod_delta(delta)
    caps = np.full(enc.T, 40, np.int32)
    for rank in (0, 1):
        a, b = Engine(device=0, rank=rank, world_size=2), Engine(device=0, rank=rank, world_size=2)
        try:
            a.load(enc)
            assert a.load_pods(delta, after) == 0
            b.load(after)
            for x, y in zip(a.estimate_all(caps), b.estimate_all(caps)):
                assert np.array_equal(x, y), rank
        finally:
            a.close()
            b.close()


def test_limits_and_overflow_leave_the_engine_unchanged(engines):
    """status 1 (> 8 topology keys, > 12 counters for one pod, the rank-encoding width) and status 2 (a table past
    2^31 - 1, a request in a dim past num_res): the outputs stay those of the load, and a later delta still applies"""
    eng, fresh = engines(False)
    enc = _gen("c3")
    eng.load(enc)
    want = _results(eng, enc)
    s = enc.struct
    sel = 0                                                   # selector 0 of the load
    n_keys = 9
    keys = PodDelta(pts_off=np.arange(n_keys + 1), pts_max_skew=np.ones(n_keys), pts_key=10_000 + np.arange(n_keys),
                    pts_selector=np.full(n_keys, sel), pts_min_domains=np.ones(n_keys), pts_node_affinity_policy=np.ones(n_keys),
                    pts_node_taints_policy=np.zeros(n_keys),
                    **_new_specs(enc, n_keys, ps_pts_list=s.num_pts_lists + np.arange(n_keys)))
    m = 13
    counters = PodDelta(pts_off=[0, m], pts_max_skew=np.ones(m), pts_key=np.full(m, 10_000), pts_selector=np.full(m, sel),
                        pts_min_domains=np.ones(m), pts_node_affinity_policy=np.ones(m), pts_node_taints_policy=np.zeros(m),
                        **_new_specs(enc, 1, ps_pts_list=[s.num_pts_lists]))
    n = 2100                                                  # 3 dims x 12 bit slices > 32
    req = np.zeros((n, 8), np.int64)
    req[:, :3] = 1 + np.arange(n)[:, None] * np.array([1, 3, 5])
    width = PodDelta(**_new_specs(enc, n, ps_req=req))
    for d in (keys, counters, width):
        assert eng.load_pods(d) == 1
    big = _synth_delta(enc, 5, 2)
    big.struct.num_new_values = 2**31 - 1                     # checked from the count before any value is read
    assert eng.load_pods(big) == 2
    req = np.repeat(enc.arrays["ps_req"][:1], 1, axis=0)
    req[0, 7] = 1
    assert eng.load_pods(PodDelta(**_new_specs(enc, 1, ps_req=req))) == 2
    _assert_same(_results(eng, enc), want, "after refusals")
    ok = _synth_delta(enc, 6, 4)
    after = enc.apply_pod_delta(ok)
    assert eng.load_pods(ok, after) == 0
    fresh.load(after)
    _assert_same(_results(eng, after), _results(fresh, after), "after a good delta")
