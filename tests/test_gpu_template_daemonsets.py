"""cae_template_daemonsets on the GPU.  The verdicts equal daemonset.py's host mirror: on the hand-worked object cases, on
random templates and DaemonSet specs (T up to 300, D = 0, 1, 31, 32, 33 and 200, with evaluate and running masks) and on
the C3 and C5 synthetic templates with 50 DaemonSets.  After an apply, every entry point answers as an engine that got the
host-built lists through cae_load_templates, as a fresh load of the resulting objects and as the oracle; also after
cae_load_pods, cae_force_add_pods and cae_load_node_churn.  Refusals (-2 and 2) leave every answer unchanged, and ranks of
worlds of 2 to 8 answer alike."""
import numpy as np
import pytest

from delta_harness import SHAPES, _assert_same, _check, _gen, _results, engines  # noqa: F401  (engines: fixture)
from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.daemonset import (NodeShouldRunDaemonPod, apply_run_bits, pack_rows, run_bits_encoded,
                                                  unpack_rows)

pytestmark = pytest.mark.gpu


def _used_specs(enc):
    """Specs some pending or resident pod has: a DaemonSet of one of them is never refused for anti-affinity."""
    a = enc.arrays
    return np.unique(np.concatenate([a["pend_spec"], a["node_pod_spec"]])).astype(np.int32)


def _draw(enc, seed, D, masks=True):
    rng = np.random.default_rng(seed)
    T = enc.T
    ds = rng.integers(0, enc.struct.num_podspecs, D).astype(np.int32)
    ev = (rng.random(T) < 0.8).astype(np.uint8) if masks else None
    run = rng.random((T, D)) < 0.2 if masks else None
    return ds, ev, run


def _verdicts_equal(eng, enc, ds, ev=None, run=None):
    D = len(ds)
    bits, count = eng.template_daemonsets(ds, ev, None if run is None else pack_rows(run, D))
    want = run_bits_encoded(enc, ds, ev, run)
    assert bits.shape == (enc.T, (D + 31) // 32)
    assert np.array_equal(unpack_rows(bits, D), want)
    assert np.array_equal(count, want.sum(axis=1))
    if D % 32:   # padding bits of the last word stay 0
        assert not (bits[:, -1] >> (D % 32)).any()
    return want


def test_hand_worked_cases(engines):
    from test_template_daemonsets_host import CASES, _encoded
    from kubernetes_autoscaler_b200.objects import NodeInfo
    eng, _ = engines(False)
    nodes = [c[1] for c in CASES]
    dss = [c[2] for c in CASES]
    _, enc, ids = _encoded([NodeInfo(n, []) for n in nodes], dss)
    eng.load(enc)
    want = np.array([[NodeShouldRunDaemonPod(n, ds)[0] for ds in dss] for n in nodes])
    assert np.array_equal(_verdicts_equal(eng, enc, ids), want)
    for c, (case, *_rest, w) in enumerate(CASES):   # the diagonal is each case's own verdict
        assert want[c, c] == w, case


@pytest.mark.parametrize("D", [0, 1, 31, 32, 33, 200])
@pytest.mark.parametrize("T", [1, 33, 300])
def test_random_templates_and_daemonsets(engines, T, D):
    eng, _ = engines(False)
    enc = synth.generate(2, pods=300, templates=T, cluster_nodes=16, seed=T * 1000 + D)
    eng.load(enc)
    ds, ev, run = _draw(enc, T + D, D)
    _verdicts_equal(eng, enc, ds, ev, run)
    _verdicts_equal(eng, enc, ds)
    bits, count = eng.template_daemonsets(ds, np.zeros(T, np.uint8))
    assert not bits.any() and not count.any()


@pytest.mark.parametrize("config", [3, 5])
def test_synth_templates_with_50_daemonsets(engines, config):
    eng, _ = engines(False)
    enc = synth.generate(config, pods=2000)
    eng.load(enc)
    ds, ev, run = _draw(enc, config, 50)
    want = _verdicts_equal(eng, enc, ds)
    assert want.any() and not want.all(), "the shapes exercise both verdicts"
    _verdicts_equal(eng, enc, ds, ev, run)


def _similar(eng, enc):
    from test_gpu_template_delta import _similar as sim
    return sim(eng, enc)


def _apply_case(enc, seed, D=24):
    rng = np.random.default_rng(seed)
    N, T = enc.struct.num_cluster_nodes, enc.T
    used = _used_specs(enc)
    ds = used[rng.integers(0, len(used), D)]
    off = enc.arrays["node_pod_off"]
    pods = off[N + 1:N + T + 1] - off[N:N + T]
    keep = (rng.random(T) * (pods + 1)).astype(np.int32)
    keep[::4] = pods[::4]
    ev = (rng.random(T) < 0.85).astype(np.uint8)
    run = rng.random((T, D)) < 0.1
    return ds, ev, run, keep


def _apply_and_check(eng, twin, fresh, oracle, cur, seed, with_oracle):
    """`eng` holds `cur`: apply on it, and the host-built lists on `twin` (also holding `cur`) through cae_load_templates."""
    ds, ev, run, keep = _apply_case(cur, seed)
    bits, count = eng.template_daemonsets(ds, ev, pack_rows(run, len(ds)), keep)
    want = run_bits_encoded(cur, ds, ev, run)
    assert np.array_equal(unpack_rows(bits, len(ds)), want)
    delta, after = apply_run_bits(cur, ds, want, keep, ev)
    assert delta.num_changed > 0
    assert twin.load_templates(delta, after)
    got = _check(eng, fresh, oracle, after, True, with_oracle=with_oracle)
    _assert_same(_results(twin, after), got, "cae_load_templates of the host-built lists")
    for x, y in zip(_similar(eng, after), _similar(twin, after)):
        assert np.array_equal(x, y), "similar node groups differ"
    return after


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_apply_matches_template_delta_and_full_load(engines, oracle, shape):
    from kubernetes_autoscaler_b200.engine import Engine
    eng, fresh = engines(True)
    twin = Engine(device=0, want_reasons=True)
    try:
        enc = _gen(shape)
        eng.load(enc)
        twin.load(enc)
        after = _apply_and_check(eng, twin, fresh, oracle, enc, 11, True)
        # a second apply on the result, and one with no DaemonSet: every evaluated template stripped to its prefix
        after = _apply_and_check(eng, twin, fresh, oracle, after, 12, False)
        keep = np.zeros(after.T, np.int32)
        eng.template_daemonsets(np.zeros(0, np.int32), None, None, keep)
        delta, stripped = apply_run_bits(after, np.zeros(0, np.int32), np.zeros((after.T, 0), bool), keep)
        assert twin.load_templates(delta, stripped)
        assert stripped.arrays["node_pod_off"][-1] == stripped.arrays["node_pod_off"][stripped.struct.num_cluster_nodes]
        got = _check(eng, fresh, oracle, stripped, True, with_oracle=False)
        _assert_same(_results(twin, stripped), got, "cae_load_templates of the stripped lists")
    finally:
        twin.close()


@pytest.mark.parametrize("shape", ["c3", "c4"])
def test_apply_after_other_deltas(engines, oracle, shape):
    from kubernetes_autoscaler_b200.engine import Engine
    eng, fresh = engines(True)
    twin = Engine(device=0, want_reasons=True)
    try:
        cur = _gen(shape)
        eng.load(cur)
        pd = synth.pod_churn(cur, 71, 3, 2)
        cur = cur.apply_pod_delta(pd)
        assert eng.load_pods(pd, cur) == 0
        twin.load(cur)
        cur = _apply_and_check(eng, twin, fresh, oracle, cur, 21, False)
        N = cur.struct.num_cluster_nodes
        pods = np.arange(0, min(cur.P, 40), 8)
        nodes = np.arange(len(pods)) % max(N, 1)
        cur, _ = cur.apply_force_add(pods, nodes)
        assert eng.force_add_pods(pods, nodes, cur) is not False
        twin.load(cur)
        cur = _apply_and_check(eng, twin, fresh, oracle, cur, 22, False)
        churn, pending = synth.node_scale(cur, 73, 2, 2, 3)
        assert eng.load_node_churn(churn) and eng.load_pending(pending)
        cur = pending.apply_node_churn(churn)
        twin.load(cur)
        _apply_and_check(eng, twin, fresh, oracle, cur, 23, True)
    finally:
        twin.close()


def test_refusals_leave_every_answer_unchanged(engines):
    from test_gpu_node_churn import _anti_world
    from kubernetes_autoscaler_b200.engine import EngineError, EngineUnsupported
    from kubernetes_autoscaler_b200.encode import DaemonSetInputs
    eng, _ = engines(False)
    enc = _gen("c3")
    eng.load(enc)
    before = _results(eng, enc)
    T, S = enc.T, enc.struct.num_podspecs
    pods = np.diff(enc.arrays["node_pod_off"][enc.struct.num_cluster_nodes:])
    ds = np.resize(_used_specs(enc), 33)   # two words, the second ragged
    bad = {
        "spec out of range": dict(ds_spec=np.r_[ds[:-1], S]),
        "negative spec": dict(ds_spec=np.r_[-1, ds[1:]]),
        "evaluate byte": dict(ds_spec=ds, evaluate=np.full(T, 2, np.uint8)),
        "running past num_ds": dict(ds_spec=ds, running=np.tile(np.array([0, 1 << 1], np.uint32), (T, 1))),
        "keep < 0": dict(ds_spec=ds, keep=np.r_[-1, np.zeros(T - 1, np.int32)]),
        "keep past the pods": dict(ds_spec=ds, keep=(pods + 1).astype(np.int32)),
    }
    for what, kw in bad.items():
        with pytest.raises(EngineError):
            eng.template_daemonsets(**kw)
        _assert_same(_results(eng, enc), before, "after a refused call (%s)" % what)
    di = DaemonSetInputs(ds_spec=ds)
    di.struct.num_ds = -1
    assert eng.lib.cae_template_daemonsets(eng.h, di.ptr(), None, None) == -2
    di = DaemonSetInputs(ds_spec=ds)
    di.struct.ds_spec = None
    assert eng.lib.cae_template_daemonsets(eng.h, di.ptr(), None, None) == -2
    _assert_same(_results(eng, enc), before, "after refused structs")
    # status 2: a DaemonSet spec with anti-affinity terms that no pod of the snapshot had
    _, enc2, _, _ = _anti_world()
    eng.load(enc2)
    before2 = _results(eng, enc2)
    lonely = np.array([enc2.struct.num_podspecs - 1], np.int32)
    assert enc2.arrays["ps_anti_list"][lonely[0]] != 0
    bits, _ = eng.template_daemonsets(lonely)
    assert bits.any(), "the lonely spec runs somewhere"
    with pytest.raises(EngineUnsupported):
        eng.template_daemonsets(lonely, keep=np.diff(enc2.arrays["node_pod_off"][enc2.struct.num_cluster_nodes:]).astype(np.int32))
    _assert_same(_results(eng, enc2), before2, "after a refused apply")


def test_ranks_answer_alike(engines):
    from kubernetes_autoscaler_b200.engine import Engine
    one, _ = engines(False)
    enc = _gen("c2")
    ds, ev, run, keep = _apply_case(enc, 31)
    want_bits, want_count = None, None
    one.load(enc)
    want_bits, want_count = one.template_daemonsets(ds, ev, pack_rows(run, len(ds)), keep)
    after = one.enc
    caps = np.full(after.T, 30, np.int32)
    want_est = one.estimate_all(caps)
    for W in range(2, 9):
        got = [np.zeros(after.T, np.int32) for _ in range(3)]
        for r in range(W):
            e = Engine(device=0, rank=r, world_size=W)
            try:
                e.load(enc)
                bits, count = e.template_daemonsets(ds, ev, pack_rows(run, len(ds)), keep)
                assert np.array_equal(bits, want_bits) and np.array_equal(count, want_count), (W, r)
                est = e.estimate_all(caps)
                for i in range(2):
                    got[i] += est[i]
                got[2] += est[2].sum(axis=1) if est[2] is not None else 0
            finally:
                e.close()
        assert np.array_equal(got[0], want_est[0]) and np.array_equal(got[1], want_est[1]), W
        assert np.array_equal(got[2], want_est[2].sum(axis=1)), W
