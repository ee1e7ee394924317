"""Shared helpers of the GPU delta tests (cae_load_nodes, cae_load_node_churn, cae_load_pods): the synthetic shapes, a pair
of engines per reasons setting (the one under test and one for fresh loads), everything the entry points answer for a
loaded snapshot, the same from the oracle, and the comparison of both."""
import numpy as np
import pytest

from kubernetes_autoscaler_b200 import synth

SHAPES = {
    "c2": (2, dict(pods=3000, templates=40, cluster_nodes=48)),      # taints, tolerations, nodeSelectors
    "c3": (3, dict(pods=2500, templates=24, cluster_nodes=48)),      # zone / hostname spread, minDomains
    "c4": (4, dict(pods=3000, templates=20, cluster_nodes=40)),      # + anti-affinity and affinity
}


@pytest.fixture(scope="module")
def engines():
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    made = {}

    def get(reasons: bool):
        if reasons not in made:
            made[reasons] = (Engine(device=0, want_reasons=reasons), Engine(device=0, want_reasons=reasons))
        return made[reasons]
    yield get
    for a, b in made.values():
        a.close()
        b.close()


def _gen(shape, **over):
    cfg, kw = SHAPES[shape]
    return synth.generate(cfg, **{**kw, **over})


def _filter_args(enc, last=11):
    P, N = enc.P, enc.struct.num_cluster_nodes
    n = min(P, 700)
    order = np.arange(n, dtype=np.int32)[::-1].copy()
    rng = synth.SplitMix64(0xF17E)
    hint = np.where(rng.uniform(P) < 0.1, rng.randint(P, max(N, 1)), -1).astype(np.int32)
    cls = np.where(rng.uniform(P) < 0.5, rng.randint(P, 6), -1).astype(np.int32)
    ctrl = np.array([0, 1, 1, 2, 3, 3], np.int32)
    return order, hint, cls, ctrl, None, last


def _prices(enc):
    node_price = 1.0 + np.arange(enc.T, dtype=np.float64) * 0.37
    pod_price = 0.01 + (np.arange(enc.struct.num_podspecs, dtype=np.float64) % 13) * 0.003
    return node_price, pod_price


def _results(eng, enc):
    """Everything the entry points answer for the loaded snapshot (engine `eng`, shapes of `enc`)."""
    from kubernetes_autoscaler_b200.engine import unpack_bits
    eng.enc = enc
    out = {}
    bits, reasons, count = eng.feasibility()
    out["bits"] = unpack_bits(bits, enc.P).copy()
    out["count"] = count.copy()
    if reasons is not None:
        out["reasons"] = reasons.copy()
    out["groups"] = eng.feasibility_groups()
    T, N = enc.T, enc.struct.num_cluster_nodes
    node_price, pod_price = _prices(enc)
    for cap in (40, 0):
        caps = np.full(T, cap, np.int32)
        nc, pc, sched, order = eng.estimate_all(caps)
        out["est%d" % cap] = (nc, pc, sched, order)
        out["waste%d" % cap] = eng.waste_scores()
        out["best%d" % cap] = eng.expander_best([0, 1, 2], nc, pc)
        out["price%d" % cap] = eng.price_scores(node_price, pod_price, 0.5, 1500)
    li = (np.arange(T, dtype=np.int32) * 37 + 3 * N + 5).astype(np.int32)     # RAW: larger than the node list
    out["li"] = eng.estimate_all_li(np.full(T, 25, np.int32), li)
    out["filter"] = eng.filter_schedulable(*_filter_args(enc))
    out["filter_raw"] = eng.filter_schedulable(*_filter_args(enc, last=7 * N + 3))
    return out


def _oracle_results(oracle, enc, want_reasons):
    out = {}
    reasons, _ = oracle.feasibility_dense(enc)
    out["bits"] = reasons == 0
    out["count"] = (reasons == 0).sum(axis=1).astype(np.int32)
    if want_reasons:
        out["reasons"] = reasons
    out["groups"] = oracle.feasibility_groups(enc)
    T, N = enc.T, enc.struct.num_cluster_nodes
    node_price, pod_price = _prices(enc)
    for cap in (40, 0):
        caps = np.full(T, cap, np.int32)
        nc, pc, sched, order, _ = oracle.estimate_all(enc, caps)
        out["est%d" % cap] = (nc, pc, sched, order)
        mask, waste = oracle.expander(enc, [0, 1, 2], nc, pc, sched)
        out["waste%d" % cap] = waste
        out["best%d" % cap] = (mask, waste)
        out["price%d" % cap] = oracle.price_scores(enc, node_price, pod_price, 0.5, 1500, node_count=nc, sched=sched, order=order)
    li = (np.arange(T, dtype=np.int32) * 37 + 3 * N + 5).astype(np.int32)
    out["li"] = oracle.estimate_all_li(enc, np.full(T, 25, np.int32), li)
    order, hint, cls, ctrl, ok, last = _filter_args(enc)
    out["filter"] = oracle.filter_schedulable(enc, order, hint, cls, ctrl, ok, last)
    return out


def _equal(x, y):
    if isinstance(x, tuple):
        return len(x) == len(y) and all(_equal(a, b) for a, b in zip(x, y))
    if isinstance(x, np.ndarray) or isinstance(y, np.ndarray):
        return np.array_equal(np.asarray(x), np.asarray(y))
    return x == y


def _assert_same(got, want, what):
    for k in want:
        assert _equal(got[k], want[k]), "%s: %s differs" % (what, k)


def _check(eng, fresh, oracle, after, want_reasons, with_oracle=True):
    """`eng` holds `after` through deltas: compare with a fresh cae_load of `after` and (optionally) with the oracle."""
    got = _results(eng, after)
    fresh.load(after)
    _assert_same(got, _results(fresh, after), "fresh load")
    if with_oracle:
        _assert_same(got, _oracle_results(oracle, after, want_reasons), "oracle")
    return got
