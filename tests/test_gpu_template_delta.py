"""cae_load_templates on the GPU: after node-group templates are removed, changed and added, every entry point answers
bit-identically to a second engine freshly loaded with EncodedObjects.apply_template_delta(...), and to the oracle where
that is affordable — dense bits / reasons / counts, group reasons, Estimate() (capped, unlimited, RAW lastIndex), waste
and price scores, the filter-out-schedulable pass — and cae_similar_node_groups answers like the fresh engine.  Covered:
each kind of change alone and together, a DaemonSet rollout, a name-only change, zone values that move or appear, T -> 0,
0 -> T, T crossing 32 and 512 (the template words and their pitch change), ten template deltas chained with the other
delta calls, the estimate shards of two ranks, and every refusal and malformed input with the engine left as it was."""
import numpy as np
import pytest

from delta_harness import SHAPES, _assert_same, _check, _gen, _results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.encode import NodeDelta, TemplateDelta

pytestmark = pytest.mark.gpu

KINDS = {"changed": (5, 0, 0), "removed": (0, 4, 0), "added": (0, 0, 5), "all": (6, 4, 5), "new-zone": (1, 0, 0)}


def _similar(eng, enc):
    T = enc.T
    res_sig = (np.arange(T) % 3).astype(np.int32)
    free_dims = np.full(T, 0b11, np.uint32)
    return eng.similar_node_groups(res_sig, free_dims, np.ones(T, np.uint8), 10 + np.arange(T) % 5, np.arange(T) % 3,
                                   np.array([synth.K_HOST, synth.K_ZONE], np.int32), None, (0.05, 0.05, 0.015))


def _check_all(eng, fresh, oracle, after, want_reasons, with_oracle):
    _check(eng, fresh, oracle, after, want_reasons, with_oracle=with_oracle)
    if after.T:
        got, want = _similar(eng, after), _similar(fresh, after)   # fresh holds `after` after _check
        for x, y in zip(got, want):
            assert np.array_equal(x, y), "similar node groups differ"


def _all_rows(enc):
    """A delta that adds every template of `enc` (to an engine that holds none)."""
    return synth._template_delta(enc, {}, [], [], synth._template_rows(enc, range(enc.T)))


def _drop_all(enc):
    return TemplateDelta(removed=np.arange(enc.T))


@pytest.mark.parametrize("want_reasons", [False, True], ids=["bits", "reasons"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_template_delta_matches_full_load(engines, oracle, shape, want_reasons):
    eng, fresh = engines(want_reasons)
    enc = _gen(shape)
    for k, (kind, (nc, nr, na)) in enumerate(sorted(KINDS.items())):
        delta = synth.template_churn(enc, 21 + k, nc, nr, na)
        after = enc.apply_template_delta(delta)
        eng.load(enc)
        assert eng.load_templates(delta, after), kind
        _check_all(eng, fresh, oracle, after, want_reasons, with_oracle=want_reasons)
    # a DaemonSet rollout: every template's pod list changes
    roll = synth.daemonset_rollout(enc, 3)
    after = enc.apply_template_delta(roll)
    eng.load(enc)
    assert eng.load_templates(roll, after)
    _check_all(eng, fresh, oracle, after, want_reasons, with_oracle=True)
    # a name-only change (the provider's random suffix)
    rows = synth._template_rows(enc, [1])
    rows["name"][0] = int(enc.arrays["node_name"].max()) + 7
    named = synth._template_delta(enc, {}, [], [1], rows)
    after = enc.apply_template_delta(named)
    eng.load(enc)
    assert eng.load_templates(named, after)
    _check_all(eng, fresh, oracle, after, want_reasons, with_oracle=False)
    # T -> 0, then 0 -> T
    empty = enc.apply_template_delta(_drop_all(enc))
    eng.load(enc)
    assert eng.load_templates(_drop_all(enc), empty)
    _check(eng, fresh, oracle, empty, want_reasons, with_oracle=False)
    back = _all_rows(enc)
    assert eng.load_templates(back, empty.apply_template_delta(back))
    _check_all(eng, fresh, oracle, empty.apply_template_delta(back), want_reasons, with_oracle=False)


@pytest.mark.parametrize("shape", ["c2", "c4"])
def test_template_count_crosses_word_and_pitch_bounds(engines, oracle, shape):
    """T crossing 32 (a second template word) and 512 (the pitch Twp grows from 16 to 32 words), in both directions"""
    eng, fresh = engines(True)
    for T0, na, nr in ((24, 20, 0), (40, 0, 12), (500, 30, 0), (530, 0, 40)):
        enc = _gen(shape, templates=T0, pods=1500)
        delta = synth.template_churn(enc, T0, 2, nr, na)
        after = enc.apply_template_delta(delta)
        assert (T0 - 1) // 32 != (after.T - 1) // 32
        eng.load(enc)
        assert eng.load_templates(delta, after)
        _check_all(eng, fresh, oracle, after, True, with_oracle=T0 < 100)


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_ten_chained_template_deltas(engines, oracle, shape):
    """template deltas interleaved with cae_load_nodes, cae_load_node_churn, cae_load_pods, cae_load_pending and
    cae_force_add_pods, the template delta first and last by turns"""
    eng, fresh = engines(True)
    cur = _gen(shape)
    eng.load(cur)
    for k in range(10):
        tdelta = synth.template_churn(cur, 400 + k, 1 + k % 3, k % 3, 1 + (k * 2) % 4)
        if k % 2 == 0:
            cur = cur.apply_template_delta(tdelta)
            assert eng.load_templates(tdelta, cur)
        if k % 3 == 0:
            churn, pending = synth.node_scale(cur, 500 + k, 1 + k % 2, 2, 3)
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
            cur = pending.apply_node_churn(churn)
        elif k % 3 == 1:
            delta, pending = synth.node_churn(cur, 600 + k, 4)
            assert eng.load_pending(pending) and eng.load_nodes(delta)
            cur = pending.apply_node_delta(delta)
        else:
            pd = synth.pod_churn(cur, 700 + k, 2, 1)
            cur = cur.apply_pod_delta(pd)
            assert eng.load_pods(pd, cur) == 0
        if k % 4 == 3:
            N = cur.struct.num_cluster_nodes
            pods = np.arange(0, min(cur.P, 40), 8)
            nodes = np.arange(len(pods)) % max(N, 1)
            cur, _ = cur.apply_force_add(pods, nodes)
            assert eng.force_add_pods(pods, nodes, cur) is not False
        if k % 2 == 1:
            tdelta = synth.template_churn(cur, 400 + k, 1 + k % 3, k % 3, 1 + (k * 2) % 4)
            cur = cur.apply_template_delta(tdelta)
            assert eng.load_templates(tdelta, cur)
        _check(eng, fresh, oracle, cur, True, with_oracle=k in (4, 9))


def test_two_ranks_sum_to_one_engine(engines):
    """world_size 2 (two engines on one device): after a delta that changes T, the estimate shards sum to the result of one
    engine"""
    from kubernetes_autoscaler_b200.engine import Engine
    _, fresh = engines(False)
    enc = _gen("c3")
    delta = synth.template_churn(enc, 9, 3, 2, 7)
    after = enc.apply_template_delta(delta)
    fresh.load(after)
    caps = np.full(after.T, 30, np.int32)
    want = fresh.estimate_all(caps)
    ranks = [Engine(device=0, rank=r, world_size=2) for r in range(2)]
    try:
        got = []
        for e in ranks:
            e.load(enc)
            assert e.load_templates(delta, after)
            got.append(e.estimate_all(caps))
        for i in range(3):   # node_count, pod_count, sched
            assert np.array_equal(np.asarray(got[0][i]) + np.asarray(got[1][i]), np.asarray(want[i])), i
    finally:
        for e in ranks:
            e.close()


def test_refusals_leave_the_engine_unchanged(engines):
    from test_gpu_node_churn import _anti_world
    eng, _ = engines(False)
    enc = _gen("c3")
    eng.load(enc)
    before = _results(eng, enc)
    ok = synth.template_churn(enc, 4, 3, 2, 3)
    huge_rows = ok.replace()
    huge_rows.struct.num_removed = 0
    huge_rows.struct.num_changed = 0
    huge_rows.struct.num_added = 2 ** 30 - enc.struct.num_cluster_nodes // 2   # N + 2T' > 2^31 - 1; no row is read
    huge_dict = ok.replace(tails=ok.tails.replace())
    huge_dict.tails.struct.num_new_values = 2 ** 31 - enc.struct.num_values
    alloc = ok.arrays["alloc"].copy()
    alloc[:, enc.struct.num_res] = 1                                           # a dim past the load's num_res
    past = ok.replace(alloc=alloc)
    refused = {
        "template rows": huge_rows,
        "resident pods": ok.replace(pod_off=np.array([0, 1, 2, 3, 4, 5, 2 ** 31 - 64], np.int32), pod_spec=[0] * 5),
        "dictionary": huge_dict,
        "dim past num_res": past,
    }
    assert enc.struct.num_res < 8
    for what, d in refused.items():
        assert not eng.load_templates(d), what
        _assert_same(_results(eng, enc), before, "after a refused delta (%s)" % what)
    # a template pod whose anti-affinity spec was in no pod of the last load
    enc_w, enc2, cluster, lonely = _anti_world()
    eng.load(enc2)
    before2 = _results(eng, enc2)
    d = synth._template_rows(enc2, [0])
    d["pods"][0] = [enc2.struct.num_podspecs - 1]
    assert not eng.load_templates(synth._template_delta(enc2, {}, [], [], d))
    _assert_same(_results(eng, enc2), before2, "after a refused anti-affinity template pod")


def test_malformed_template_deltas(engines):
    from kubernetes_autoscaler_b200.engine import EngineError
    eng, _ = engines(False)
    enc = _gen("c2")
    T, S = enc.T, enc.struct.num_podspecs
    eng.load(enc)
    before = _results(eng, enc)
    ok = synth.template_churn(enc, 4, 3, 2, 3)
    rem, chg = ok.arrays["removed"], ok.arrays["changed"]
    nl = enc.struct.num_labelsets + ok.tails.struct.num_new_labelsets
    nrow = len(ok.arrays["name"])
    bad = {
        "removed out of range": ok.replace(removed=[rem[0], T]),
        "removed negative": ok.replace(removed=[-1, rem[1]]),
        "removed not increasing": ok.replace(removed=rem[::-1].copy()),
        "changed out of range": ok.replace(changed=[chg[0], chg[1], T]),
        "changed not increasing": ok.replace(changed=chg[::-1].copy()),
        "changed and removed": ok.replace(changed=sorted([int(rem[0]), int(chg[1]), int(chg[2])])),
        "label set": ok.replace(labelset=np.full(nrow, nl, np.int32)),
        "taint list": ok.replace(taint_list=np.full(nrow, enc.struct.num_taint_lists, np.int32)),
        "name": ok.replace(name=np.full(nrow, -1, np.int32)),
        "pod spec": ok.replace(pod_off=np.concatenate([[0], np.ones(nrow, np.int32)]), pod_spec=[S]),
        "offsets start": ok.replace(pod_off=ok.arrays["pod_off"] + 1),
        "offsets decrease": ok.replace(pod_off=np.concatenate([[0, 5, 3], np.full(nrow - 2, 5, np.int32)]), pod_spec=[0] * 5),
        "dirty tails": ok.replace(tails=NodeDelta(row=[0], labelset=[0], taint_list=[0], unschedulable=[0], allowed_pods=[1],
                                                  pod_off=[0, 0])),
    }
    for field in ("name", "labelset", "taint_list", "unschedulable", "alloc", "allowed_pods", "cap_cpu", "cap_mem",
                  "has_alloc_cpu", "has_alloc_mem", "pod_off", "removed", "changed"):
        d = ok.replace()
        setattr(d.struct, field, None)
        bad["null " + field] = d
    d = ok.replace()
    d.struct.abi_version = 99
    bad["abi version"] = d
    d = ok.replace()
    d.struct.num_added = -1
    bad["negative count"] = d
    for what, d in bad.items():
        with pytest.raises(EngineError, match="status -2"):
            eng.load_templates(d)
        _assert_same(_results(eng, enc), before, "after a malformed delta (%s)" % what)
    assert eng.load_templates(TemplateDelta())
    _assert_same(_results(eng, enc), before, "after an empty delta")
