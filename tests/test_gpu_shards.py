"""Sharded engines (cae_config.rank / world_size) on one GPU, every entry point, against the oracle and a one-rank engine.

Ranks of one world are independent engines until peers are attached, so each rank runs here on its own, one at a time,
beside at most one other engine (a one-rank engine or a freshly loaded twin):

* the dense pass over pods sharded by the engine: each rank's bits, reasons and fit counts equal the oracle's columns of
  its shard, and the ranks' raw bit words, joined in rank order, equal the one-rank engine's words (padding included);
  shards that start past pod 0, empty shards on middle ranks, every pod on the last rank, P at and next to a multiple of
  32 x world_size, template words and their pitch at T = 31, 33, 513, two constraint shapes and 6 and 8 active dims;
* the same grid with presharded pods (CAE_CFG_PODS_PRESHARDED, each rank loads EncodedObjects.slice_pods of its shard):
  dense pass, exemplar reasons and cae_group_reasons on the slice, a group split over two ranks, a group this rank holds
  no pod of, and cae_force_add_pods refused;
* Estimate() over templates sharded: own rows equal the oracle's, foreign rows zero (order -1), also with a RAW
  lastIndex; ranks without a template; summed waste and price vectors bit-equal to one engine's, also after the caller
  all-reduced node_count | pod_count in place on the device; the host expander chains on the summed vectors pick one
  engine's options;
* the calls every rank answers whole (group reasons, similar node groups, scale-down eligibility, the filter pass, the
  removal and capacity batches) equal one rank's answers at every rank of three;
* a chain of deltas on every rank of three against a freshly loaded twin of the same rank, with status 2 predicted from
  the shard sizes of the last load.

The non-GPU test at the end checks that the parameters reach every one of these cases."""
import functools

import numpy as np
import pytest

import group_reasons_ref as ref
import rank_layout
from delta_harness import _equal, _filter_args, _gen, _prices
from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import TemplateDelta
from kubernetes_autoscaler_b200.engine import expander_chain, expander_chain_ex, shard_pods, shard_templates, unpack_bits

# name -> (world_size, synth config, generate() keywords)
DENSE = {
    "w2_all_on_last_rank": (2, 2, dict(pods=20, templates=50)),
    "w2_ragged": (2, 3, dict(pods=1001, templates=40, cluster_nodes=40)),
    "w3_empty_first_ranks": (3, 2, dict(pods=40, templates=40)),
    "w3_middle_past_0": (3, 3, dict(pods=1000, templates=40, cluster_nodes=40)),
    "w4_exact": (4, 2, dict(pods=1280, templates=70)),
    "w4_exact_minus_1": (4, 2, dict(pods=1279, templates=70)),
    "w4_exact_plus_1": (4, 3, dict(pods=1281, templates=70, cluster_nodes=40)),
    "w5_exact_dims6": (5, 2, dict(pods=1600, templates=45, dims=rank_layout.DIM_SETS[6])),
    "w5_dims8": (5, 2, dict(pods=2500, templates=100, dims=rank_layout.DIM_SETS[8])),
    "w7_T31": (7, 2, dict(pods=3000, templates=31)),
    "w7_T33": (7, 2, dict(pods=3000, templates=33)),
    "w7_T513": (7, 2, dict(pods=3000, templates=513)),
    "w8_empty_middle_ranks": (8, 3, dict(pods=40, templates=24, cluster_nodes=40)),
    "w8_c3": (8, 3, dict(pods=2600, templates=60, cluster_nodes=40)),
}

# Estimate(): shapes x world sizes, and the template counts of each world size
EST_SHAPES = {"c2": (2, dict(pods=1500, cluster_nodes=24)), "c3": (3, dict(pods=1000, cluster_nodes=30))}
EST_WORLDS = (2, 3, 4, 8)
CHAINS = ([0], [0, 1, 2], [2, 0], [1], [3, 2])
PRICE = 3   # CAE_EXP_PRICE: scored on the host by cae_expander_chain_ex only


def est_templates(W):
    return sorted({1, W - 1, W, W + 1, 33, 130} - {0})


def _caps(T):
    """0 (unlimited), small, 40 and a negative cap (no node may be added)"""
    return np.array([0, 3, 40, -1, 1], np.int32)[np.arange(T) % 5]


def _raw_last_index(enc):
    N = enc.struct.num_cluster_nodes
    return (np.arange(enc.T, dtype=np.int32) * 37 + 3 * N + 5).astype(np.int32)    # RAW: past the node list


def _price_args(enc):
    node_price, pod_price = _prices(enc)
    exists = (np.arange(enc.T) % 3 != 2).astype(np.uint8)
    return (node_price, pod_price, 0.5, 1500), dict(exists=exists)


def _masks(T):
    return (np.arange(T) % 3 != 1).astype(np.uint8), (np.arange(T) % 4 != 2).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def _dense_enc(name):
    _, cfg, kw = DENSE[name]
    return synth.generate(cfg, **kw)


@functools.lru_cache(maxsize=None)
def _est_enc(shape, T):
    cfg, kw = EST_SHAPES[shape]
    return synth.generate(cfg, templates=T, **kw)


def _split_groups(enc, W):
    """Groups whose pods lie in two or more pod shards of world W"""
    off = np.asarray(enc.arrays["group_off"])
    cuts = [shard_pods(enc.P, r, W) for r in range(W)]
    return [g for g in range(enc.E) if sum(b < off[g + 1] and off[g] < e for b, e in cuts) >= 2]


@pytest.fixture(scope="module")
def one():
    """The one-rank engine the sharded answers are measured against."""
    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200.engine import Engine
    e = Engine(device=0, want_reasons=True)
    yield e
    e.close()


def _engine(rank, W, **kw):
    from kubernetes_autoscaler_b200.engine import Engine
    return Engine(device=0, rank=rank, world_size=W, **kw)


_oracle_cache = {}


def _cached(key, fn):
    if key not in _oracle_cache:
        _oracle_cache[key] = fn()
    return _oracle_cache[key]


def _dense(e):
    """(bits, reasons or None, count) of this rank, copied out of the pinned buffers"""
    bits, reasons, count = e.feasibility()
    return bits.copy(), None if reasons is None else reasons.copy(), count.copy()


def _check_dense_shard(e, enc, want, want_reasons):
    """`want`: the oracle's reasons of exactly the pods this engine holds"""
    bits, reasons, count = _dense(e)
    T, Pl = want.shape
    assert bits.shape == (T, (Pl + 31) // 32)
    assert np.array_equal(unpack_bits(bits, Pl), want == 0), "bits"
    if want_reasons:
        assert np.array_equal(reasons, want), "reasons"
    assert np.array_equal(count, (want == 0).sum(axis=1)), "fit_count"
    assert np.array_equal(count, np.unpackbits(bits.view(np.uint8), axis=1).sum(axis=1)), "fit_count vs popcount"
    return bits, count


# ---- 1. dense pass, pods sharded by the engine -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("want_reasons", [True, False], ids=["reasons", "bits"])
@pytest.mark.parametrize("name", list(DENSE))
def test_dense_pass_on_pod_shards(one, oracle, name, want_reasons):
    W = DENSE[name][0]
    enc = _dense_enc(name)
    full = _cached(("dense", name), lambda: oracle.feasibility_dense(enc)[0])
    one.load(enc)
    one_bits, _, _ = _dense(one)
    words, total = [], np.zeros(enc.T, np.int64)
    for r in range(W):
        e = _engine(r, W, want_reasons=want_reasons)
        try:
            e.load(enc)
            pb, pe = shard_pods(enc.P, r, W)
            assert e.pod_shard(enc.P) == (pb, pe)
            bits, count = _check_dense_shard(e, enc, full[:, pb:pe], want_reasons)
            words.append(bits)
            total += count
        finally:
            e.close()
    assert np.array_equal(np.concatenate(words, axis=1), one_bits), "rank words joined != one engine's words"
    assert np.array_equal(total, (full == 0).sum(axis=1)), "summed fit_count != oracle histogram"


# ---- 2. dense and group answers, presharded pods -----------------------------------------------------------------------
def _check_groups(e, oracle, sub):
    """exemplar reasons and cae_group_reasons of the groups this rank holds, against the oracle on its slice"""
    assert np.array_equal(e.feasibility_groups(), oracle.feasibility_groups(sub)), "feasibility_groups"
    detail = ref.detail(sub)
    live = ref.nonempty(sub)
    for cons, ex in ((None, None),) + (_masks(sub.T),):
        sched, counts, got = e.group_reasons(cons, ex, want_detail=True)
        ws, wc = ref.reduce(detail, cons, ex, live)
        assert np.array_equal(got, detail), "group reasons detail"
        assert np.array_equal(sched, ws) and np.array_equal(counts, wc), "group reasons counts"
        assert not sched[~live].any() and not counts[~live].any() and not got[:, ~live].any(), "a group without pods here"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(DENSE))
def test_presharded_pods(oracle, name):
    W = DENSE[name][0]
    enc = _dense_enc(name)
    caps = _caps(enc.T)
    for r in range(W):
        pb, pe = shard_pods(enc.P, r, W)
        sub = enc.slice_pods(pb, pe)
        e = _engine(r, W, want_reasons=True, pods_presharded=True)
        try:
            e.load(sub)
            assert e.pod_shard(sub.P) == (0, sub.P)
            _check_dense_shard(e, sub, oracle.feasibility_dense(sub)[0], True)
            _check_groups(e, oracle, sub)
            if W == 3 and sub.P and sub.struct.num_cluster_nodes:
                before = _dense(e) + tuple(e.estimate_all(caps))
                assert e.force_add_pods([0, sub.P - 1], [0, 0]) is False
                assert "presharded" in e.lib.cae_last_error().decode()
                after = _dense(e) + tuple(e.estimate_all(caps))
                assert all(_equal(x, y) for x, y in zip(after, before)), "a refused force-add changed the engine"
        finally:
            e.close()


# ---- 3. Estimate() and the expanders, templates sharded ----------------------------------------------------------------
def _one_engine_answers(one, enc, caps):
    one.load(enc)
    nc, pc, sched, order = one.estimate_all(caps)
    args, kw = _price_args(enc)
    out = dict(est=(nc, pc, sched, order), waste=one.waste_scores(), price=one.price_scores(*args, **kw))
    out["best"] = {tuple(c): one.expander_best(c, nc, pc)[0] for c in CHAINS if PRICE not in c}
    return out


def _write_counts(e, counts):
    """What an in-place NCCL all_reduce of node_count | pod_count on cae_device_buffer 1 leaves there"""
    import torch
    ptr, nbytes = e.device_buffer(1)
    assert ptr and nbytes == counts.nbytes

    class _Wrap:
        __cuda_array_interface__ = {"shape": (counts.size,), "typestr": "<i4", "data": (ptr, False), "version": 3}
    torch.as_tensor(_Wrap(), device="cuda").copy_(torch.from_numpy(counts))
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("W", EST_WORLDS)
@pytest.mark.parametrize("shape", sorted(EST_SHAPES))
def test_estimate_and_expander_on_template_shards(one, oracle, shape, W):
    for T in est_templates(W):
        enc = _est_enc(shape, T)
        caps = _caps(T)
        onc, opc, osched, oorder, _ = _cached(("est", shape, T), lambda: oracle.estimate_all(enc, caps))
        oli = _cached(("li", shape, T), lambda: oracle.estimate_all_li(enc, caps, _raw_last_index(enc)))
        want = _one_engine_answers(one, enc, caps)
        for got, w in zip(want["est"], (onc, opc, osched, oorder)):
            assert np.array_equal(got, w)
        args, kw = _price_args(enc)
        summed = dict(nc=np.zeros(T, np.int64), pc=np.zeros(T, np.int64), sched=np.zeros((T, enc.E), np.int64),
                      order=np.full((T, enc.E), -1, np.int32), waste=np.zeros(T), price=np.zeros(T), li=np.zeros(T, np.int64))
        for r in range(W):
            tb, te = shard_templates(T, r, W)
            own = np.zeros(T, bool)
            own[tb:te] = True
            e = _engine(r, W)
            try:
                e.load(enc)
                assert e.template_shard(T) == (tb, te)
                nc, pc, sched, order = e.estimate_all(caps)     # status 0 also on a rank without templates
                for got, w, pad in ((nc, onc, 0), (pc, opc, 0), (sched, osched, 0), (order, oorder, -1)):
                    assert np.array_equal(got[own], w[own]), "own rows (T=%d, rank %d)" % (T, r)
                    assert (got[~own] == pad).all(), "foreign rows (T=%d, rank %d)" % (T, r)
                waste, price = e.waste_scores(), e.price_scores(*args, **kw)
                for got, w in ((waste, want["waste"]), (price, want["price"])):
                    assert np.array_equal(got[own], w[own]) and not got[~own].any(), "scores (T=%d, rank %d)" % (T, r)
                # the counts all-reduced in place on the device: the scores still cover this rank's rows only
                _write_counts(e, np.concatenate([onc, opc]).astype(np.int32))
                assert np.array_equal(e.waste_scores(), waste), "waste after the in-place all-reduce (T=%d, rank %d)" % (T, r)
                assert np.array_equal(e.price_scores(*args, **kw), price), "price after the in-place all-reduce (T=%d, rank %d)" % (T, r)
                for c, mask in want["best"].items():   # caller-supplied summed rows: every template is scored
                    got_mask, got_waste = e.expander_best(list(c), onc, opc, osched)
                    assert np.array_equal(got_mask, mask) and np.array_equal(got_waste, want["waste"]), c
                got = e.estimate_all_li(caps, _raw_last_index(enc))
                for g, w in zip(got, oli):
                    assert np.array_equal(g[own], w[own]), "estimate_all_li own rows (T=%d, rank %d)" % (T, r)
                    assert (g[~own] == (-1 if g is got[3] else 0)).all(), "estimate_all_li foreign rows (T=%d, rank %d)" % (T, r)
                summed["nc"] += nc
                summed["pc"] += pc
                summed["sched"] += sched
                summed["order"][own] = order[own]
                summed["waste"] += waste
                summed["price"] += price
                summed["li"] += got[4]
            finally:
                e.close()
        for k, w in (("nc", onc), ("pc", opc), ("sched", osched), ("order", oorder), ("li", oli[4])):
            assert np.array_equal(summed[k], w), k
        assert np.array_equal(summed["waste"], want["waste"]) and np.array_equal(summed["price"], want["price"])
        assert np.array_equal(summed["waste"], oracle.expander(enc, [0], onc, opc, osched)[1])
        for c in CHAINS:
            omask = oracle.expander_ex(c, onc, opc, waste=want["waste"], price=want["price"])
            got = expander_chain_ex(c, summed["nc"], summed["pc"], waste=summed["waste"], price=summed["price"])
            assert np.array_equal(got, omask), c
            if PRICE not in c:
                assert np.array_equal(expander_chain(c, summed["nc"], summed["pc"], summed["waste"]), want["best"][tuple(c)]), c


# ---- 4. the calls every rank answers whole -----------------------------------------------------------------------------
def _similar(e, enc):
    T = enc.T
    res_sig = (np.arange(T) % 3).astype(np.int32)
    return e.similar_node_groups(res_sig, np.full(T, 0b11, np.uint32), np.ones(T, np.uint8), 10 + np.arange(T) % 5,
                                 np.arange(T) % 3, np.array([synth.K_HOST, synth.K_ZONE], np.int32), None, (0.05, 0.05, 0.015))


def _whole_answers(e, enc):
    N, P = enc.struct.num_cluster_nodes, enc.P
    out = {"groups": e.feasibility_groups()}
    out["reasons"] = e.group_reasons(*_masks(enc.T), want_detail=True)
    out["reasons_all"] = e.group_reasons()
    out["similar"] = _similar(e, enc)
    out["eligibility"] = e.scale_down_eligibility(np.arange(N), np.full(N, -1), np.full(N, 0.5))
    out["filter"] = e.filter_schedulable(*_filter_args(enc))
    out["filter_raw"] = e.filter_schedulable(*_filter_args(enc, last=7 * N + 3))
    cand = np.array([0, 3, N - 1, 7, 3], np.int32)
    move_off = np.array([0, 4, 9, 9, 15, 18], np.int32)
    move_pod = (np.arange(18) * 53 % P).astype(np.int32)
    dest = (np.arange(N) % 5 != 1).astype(np.uint8)
    hint = np.where(np.arange(P) % 9 == 0, np.arange(P) % N, -1).astype(np.int32)
    for persist in (False, True):
        out["removals%d" % persist] = e.simulate_removals(cand, move_off, move_pod, dest, hint, last_index=5 * N + 2,
                                                          persist=persist)
    book, check = capi.CONST["CAE_CAPACITY_BOOK"], capi.CONST["CAE_CAPACITY_CHECK"]
    kinds = np.array([book, check, book, check, check], np.int32)
    off = np.array([0, 40, 90, 91, 300, 420], np.int32)
    req_pod = np.arange(0, 840, 2, dtype=np.int32) % P   # each pod in one request at most
    out["capacity"] = e.check_capacity(kinds, off, req_pod, hint_node=hint, last_index=N + 5)
    return out


@pytest.mark.gpu
def test_calls_every_rank_answers_whole(one, oracle):
    enc = synth.generate(3, pods=1000, templates=20, cluster_nodes=40)
    one.load(enc)
    want = _whole_answers(one, enc)
    assert np.array_equal(want["groups"], oracle.feasibility_groups(enc))
    assert _equal(want["reasons_all"][:2], ref.group_reasons(enc)[:2])
    for r in range(3):
        e = _engine(r, 3)
        try:
            e.load(enc)
            got = _whole_answers(e, enc)
            for k in want:
                assert _equal(got[k], want[k]), "%s differs on rank %d of 3" % (k, r)
        finally:
            e.close()


# ---- 5. deltas on sharded engines --------------------------------------------------------------------------------------
DELTA_W = 3
DELTA_P0, DELTA_PENDING = 960, (957, 900, 1000)   # pending lists of cae_load_pending after the first load, in order


@functools.lru_cache(maxsize=None)
def _delta_base():
    """c2 (no topology counters), 1000 pending pods in 10 groups, 5 templates"""
    return _gen("c2", pods=1000, templates=5)


def _trim(enc, P):
    """`enc` with P of its pending pods: every group keeps its first pod, the rest are taken group by group in order, so
    the group -> spec sequence stays that of `enc`"""
    off = np.asarray(enc.arrays["group_off"])
    n = np.diff(off)
    keep = np.minimum(n, 1)
    extra = P - int(keep.sum())
    for g in range(len(n)):
        add = min(int(n[g] - keep[g]), extra)
        keep[g] += add
        extra -= add
    assert extra == 0
    pend = np.concatenate([enc.arrays["pend_spec"][off[g]:off[g] + keep[g]] for g in range(len(n))])
    return enc.with_pending(pend, np.concatenate([[0], np.cumsum(keep)]))


def _shard_len(P, r):
    b, e = shard_pods(P, r, DELTA_W)
    return e - b


def _refused(cap, P, E, r):
    """status 2 of cae_load_pending on rank r; cap = (P, E, shard length) of the last cae_load or cae_load_pods"""
    return P > cap[0] or E > cap[1] or _shard_len(P, r) > cap[2]


def _caps_of(enc, r):
    return (enc.P, enc.E, _shard_len(enc.P, r))


def _force_add_count(P, caps):
    """The fewest pods whose force-add makes some ranks' shards outgrow their buffers, but not every rank's"""
    for n in range(1, 64):
        refuse = [_shard_len(P - n, r) > caps[r][2] for r in range(DELTA_W)]
        if any(refuse) and not all(refuse):
            return n, refuse
    raise AssertionError("no force-add size grows a shard")


def _after_pod_delta():
    cur = _trim(_delta_base(), DELTA_PENDING[-1])
    pd = synth.pod_churn(cur, 72, 3, 1)
    return pd, cur.apply_pod_delta(pd)


def _shard_answers(e, enc):
    e.enc = enc
    out = dict(zip(("bits", "reasons", "count"), _dense(e)))
    out["groups"] = e.feasibility_groups()
    args, kw = _price_args(enc)
    for cap in (40, 0):
        out["est%d" % cap] = e.estimate_all(np.full(enc.T, cap, np.int32))
        out["waste%d" % cap] = e.waste_scores()
        out["price%d" % cap] = e.price_scores(*args, **kw)
    return out


def _check_step(e, twin, oracle, enc, what, with_oracle):
    got = _shard_answers(e, enc)
    twin.load(enc)
    want = _shard_answers(twin, enc)
    for k in want:
        assert _equal(got[k], want[k]), "%s: %s differs from a fresh load on rank %d" % (what, k, e.rank)
    if with_oracle:
        pb, pe = shard_pods(enc.P, e.rank, DELTA_W)
        tb, te = shard_templates(enc.T, e.rank, DELTA_W)
        reasons = oracle.feasibility_dense(enc, p_range=(pb, pe))[0]
        assert np.array_equal(got["reasons"], reasons) and np.array_equal(unpack_bits(got["bits"], pe - pb), reasons == 0)
        assert np.array_equal(got["count"], (reasons == 0).sum(axis=1))
        assert np.array_equal(got["groups"], oracle.feasibility_groups(enc))
        onc, opc, osched, oorder, _ = oracle.estimate_all(enc, np.full(enc.T, 40, np.int32), t_range=(tb, te))
        for g, w in zip(got["est40"], (onc, opc, osched, oorder)):
            assert np.array_equal(g[tb:te], w), "%s: estimate rows differ from the oracle on rank %d" % (what, e.rank)


@pytest.mark.gpu
@pytest.mark.parametrize("rank", range(DELTA_W))
def test_delta_chain_on_every_rank(oracle, rank):
    import __graft_entry__ as g
    g.build()
    base = _delta_base()
    e, twin = _engine(rank, DELTA_W, want_reasons=True), _engine(rank, DELTA_W, want_reasons=True)
    try:
        cur = _trim(base, DELTA_P0)
        e.load(cur)
        cap = _caps_of(cur, rank)
        _check_step(e, twin, oracle, cur, "load", False)
        # cae_load_pending: 957 grows the last rank's shard past its load-time length, 1000 is more than the load's P
        for k, P in enumerate(DELTA_PENDING):
            cur = _trim(base, P)
            refuse = _refused(cap, cur.P, cur.E, rank)
            assert e.load_pending(cur) is not refuse, (P, rank)
            if refuse:
                e.load(cur)
                cap = _caps_of(cur, rank)
            _check_step(e, twin, oracle, cur, "load_pending %d" % P, k == 1)
        # cae_load_pods: new specs and a new pending list; the buffers are sized again
        pd, after = _after_pod_delta()
        assert e.load_pods(pd, after) == 0
        cur, cap = after, _caps_of(after, rank)
        _check_step(e, twin, oracle, cur, "load_pods", False)
        # cae_force_add_pods: a list that grows some ranks' shards past their buffers
        n, refuse = _force_add_count(cur.P, [_caps_of(cur, r) for r in range(DELTA_W)])
        N = cur.struct.num_cluster_nodes
        pods, nodes = np.arange(n) * 5 % cur.P, np.arange(n) % N
        after, _ = cur.apply_force_add(pods, nodes)
        res = e.force_add_pods(pods, nodes, after)
        assert (res is False) is refuse[rank], (n, rank)
        if refuse[rank]:
            e.load(after)
            cap = _caps_of(after, rank)
        cur = after
        _check_step(e, twin, oracle, cur, "force_add_pods", False)
        # cae_load_templates: T 5 -> 2 -> 0 -> 7, so template shards empty and fill again
        five = cur
        steps = [synth.template_churn(cur, 31, 1, 3, 0), TemplateDelta(removed=np.arange(2))]
        rows = synth._template_rows(five, [0, 1, 2, 3, 4, 0, 1])
        rows["name"][5:] = int(five.arrays["node_name"].max()) + 1 + np.arange(2)
        steps.append(synth._template_delta(five, {}, [], [], rows))
        for want_T, td in zip((2, 0, 7), steps):
            cur = cur.apply_template_delta(td)
            assert cur.T == want_T
            assert e.load_templates(td, cur)
            _check_step(e, twin, oracle, cur, "load_templates T=%d" % want_T, want_T == 7)
        # cae_load_nodes and cae_load_node_churn, each with the pending list the bound pods leave
        nd, pending = synth.node_churn(cur, 41, 6)
        assert e.load_nodes(nd)
        refuse = _refused(cap, pending.P, pending.E, rank)
        assert e.load_pending(pending) is not refuse
        cur = pending.apply_node_delta(nd)
        if refuse:
            e.load(cur)
            cap = _caps_of(cur, rank)
        _check_step(e, twin, oracle, cur, "load_nodes", False)
        churn, pending = synth.node_scale(cur, 43, 2, 3, 2)
        assert e.load_node_churn(churn)
        refuse = _refused(cap, pending.P, pending.E, rank)
        assert e.load_pending(pending) is not refuse
        cur = pending.apply_node_churn(churn)
        if refuse:
            e.load(cur)
        _check_step(e, twin, oracle, cur, "load_node_churn", False)
    finally:
        e.close()
        twin.close()


# ---- 6. without a GPU: the parameters reach their cases ----------------------------------------------------------------
def test_shard_parameters_reach_their_cases():
    empty_middle = past_0_not_last = ragged_last = split_group = False
    exact = {}
    for name, (W, _, kw) in DENSE.items():
        P = kw["pods"]
        cuts = [shard_pods(P, r, W) for r in range(W)]
        empty_middle |= any(b == e for b, e in cuts[1:-1])
        past_0_not_last |= any(b > 0 and e > b for b, e in cuts[:-1])
        ragged_last |= (cuts[-1][1] - cuts[-1][0]) % 32 != 0 and cuts[-1][0] > 0
        split_group |= bool(_split_groups(_dense_enc(name), W))
        if P < 32:
            assert all(b == e for b, e in cuts[:-1]), name       # every pod on the last rank
        exact.setdefault(W, set()).add(P % (32 * W))
    assert empty_middle and past_0_not_last and ragged_last and split_group
    assert {0, 1, 32 * 4 - 1} <= exact[4] and 0 in exact[5]
    assert set(W for W, _, _ in DENSE.values()) == {2, 3, 4, 5, 7, 8}
    Ts = {kw["templates"] for _, _, kw in DENSE.values()}
    assert {31, 33, 513} <= Ts and max(Ts) > 512
    assert {synth.CONFIGS[c].spread for _, c, _ in DENSE.values()} == {False, True}   # two constraint shapes
    for name, A in (("w5_exact_dims6", 6), ("w5_dims8", 8)):
        lay = rank_layout.layout_of(_dense_enc(name))
        assert lay["A"] == A and lay["path"] == "lut", lay
    # templates: a rank without a template at every world size
    for W in EST_WORLDS:
        assert any(b == e for T in est_templates(W) for b, e in (shard_templates(T, r, W) for r in range(W))), W
    # deltas: the load_pending steps refuse exactly on the ranks they are meant to
    base = _delta_base()
    caps = [_caps_of(_trim(base, DELTA_P0), r) for r in range(DELTA_W)]
    first = _trim(base, DELTA_PENDING[0])
    grown = [_refused(caps[r], first.P, first.E, r) for r in range(DELTA_W)]
    assert any(grown) and not all(grown)                          # a shard outgrows its buffer, not the whole list
    assert first.P < DELTA_P0
    last = _trim(base, DELTA_PENDING[-1])
    assert last.P > max(DELTA_P0, *DELTA_PENDING[:-1])            # more pods than any load: every rank refuses
    _, after = _after_pod_delta()
    n, refuse = _force_add_count(after.P, [_caps_of(after, r) for r in range(DELTA_W)])
    assert any(refuse) and not all(refuse)
