"""Shared part of tests/test_gpu_call_order.py: a catalogue of the engine's read-only calls (an argument generator driven by a
seeded rng and a runner that returns the answer as arrays), the snapshots the sequences load, and the single-call
reference engines and oracle anchors the answers are checked against.

The engine keeps state between calls (the last estimate's device rows, the group-reason cache, the estimator slab with its
slot versions, the one-block passes' shared buffers); the header promises that none of it shows in an answer.  So an answer
here depends only on (snapshot, call, arguments) and, for the three consumers of the device-resident estimate (waste,
price and expander without caller rows), on the arguments of the last estimate."""
import hashlib
import pickle
import random
import zlib

import numpy as np

import rank_layout
import test_gpu_fuzz as fuzz
from delta_harness import SHAPES
from kubernetes_autoscaler_b200 import capi, synth
from kubernetes_autoscaler_b200.encode import Encoder, encode
from utilization_ref import same_bits

C = capi.CONST
CHAIN = [0, 1, 2]


# ---- the arguments ---------------------------------------------------------------------------------------------------
def _sizes(enc):
    return enc.P, enc.T, enc.E, enc.struct.num_cluster_nodes


def _n_res(enc):
    N = enc.struct.num_cluster_nodes
    return int(enc.arrays["node_pod_off"][N])


def _caps(rng, T, kind=None):
    kind = kind or rng.choice(["zero", "small", "mixed", "negative", "forty"])
    if kind == "zero":
        return np.zeros(T, np.int32)
    if kind == "small":
        return rng.integers(1, 4, T).astype(np.int32)
    if kind == "negative":
        return np.full(T, -1, np.int32)
    if kind == "forty":
        return np.full(T, 40, np.int32)
    return rng.choice(np.array([-1, 0, 0, 1, 3, 8, 40], np.int32), T)


def _mask(rng, n, p=0.7):
    return None if rng.random() < 0.3 else (rng.random(n) < p).astype(np.uint8)


def _hints(rng, P, N):
    if N == 0 or rng.random() < 0.3:
        return None
    return np.where(rng.random(P) < 0.15, rng.integers(0, N, P), -1).astype(np.int32)


def _classes(rng, P):
    if rng.random() < 0.3:
        return None, None
    return np.where(rng.random(P) < 0.5, rng.integers(0, 6, P), -1).astype(np.int32), np.array([0, 1, 1, 2, 3, 3], np.int32)


def _prices(enc):
    node_price = 1.0 + np.arange(enc.T, dtype=np.float64) * 0.37
    pod_price = 0.01 + (np.arange(enc.struct.num_podspecs, dtype=np.float64) % 13) * 0.003
    return node_price, pod_price


def _caller_rows(rng, enc):
    """node_count, pod_count, sched_count, order of a caller's option table: in range for every index the kernels read."""
    P, T, E, N = _sizes(enc)
    size = np.diff(np.asarray(enc.arrays["group_off"], np.int64))
    sched = np.zeros((T, E), np.int32)
    order = np.full((T, E), -1, np.int32)
    for t in range(T):
        gs = rng.permutation(E)[:int(rng.integers(0, E + 1))]
        order[t, :len(gs)] = gs
        sched[t, gs] = (rng.random(len(gs)) * (size[gs] + 1)).astype(np.int32)
    nc = np.where(sched.sum(axis=1) > 0, rng.integers(1, 5, T), 0).astype(np.int32)
    return nc, sched.sum(axis=1).astype(np.int32), sched, order


def _split(rng, items, parts):
    """items cut into `parts` consecutive runs of random lengths (offsets, flat list)"""
    cuts = np.sort(rng.integers(0, len(items) + 1, max(parts - 1, 0)))
    return np.concatenate([[0], cuts, [len(items)]]).astype(np.int32), np.asarray(items, np.int32)


def g_feasibility(rng, enc):
    return dict(bits=bool(rng.random() < 0.7), reasons=bool(rng.random() < 0.7))


def g_none(rng, enc):
    return {}


def g_group_reasons(rng, enc, bad=False):
    T = enc.T
    cons, ex = _mask(rng, T), _mask(rng, T)
    if bad:
        cons = np.ones(T, np.uint8)
        cons[int(rng.integers(0, T))] = 2
    return dict(cons=cons, ex=ex, detail=bool(rng.random() < 0.5))


def g_estimate(rng, enc):
    return dict(caps=_caps(rng, enc.T))


def g_estimate_ex(rng, enc, bad=False):
    P, T, E, N = _sizes(enc)
    li = (rng.integers(0, 4 * max(N, 1) + 7, T)).astype(np.int32)   # RAW: up to past the node list
    if bad:
        li[int(rng.integers(0, T))] = -1
    return dict(caps=_caps(rng, T), li=li)


def g_price(rng, enc):
    return dict(stab=float(rng.choice([0.0, 0.5, 2.0])), cpu=int(rng.choice([0, 1500, 4000])),
                exists=_mask(rng, enc.T, 0.8), has_gpu=None if rng.random() < 0.6 else (rng.random(enc.T) < 0.2).astype(np.uint8))


def g_price_rows(rng, enc):
    nc, pc, sched, order = _caller_rows(rng, enc)
    return dict(g_price(rng, enc), nc=nc, sched=sched, order=order)


def g_expander(rng, enc):
    nc, pc, sched, order = _caller_rows(rng, enc)
    return dict(chain=list(rng.permutation(3)[:int(rng.integers(1, 4))]), nc=nc, pc=pc)


def g_expander_rows(rng, enc):
    nc, pc, sched, order = _caller_rows(rng, enc)
    return dict(chain=list(rng.permutation(3)[:int(rng.integers(1, 4))]), nc=nc, pc=pc, sched=sched)


def g_filter(rng, enc, n_pods=None):
    P, T, E, N = _sizes(enc)
    n = int(n_pods if n_pods is not None else rng.integers(0, min(P, 700) + 1))
    cls, ctrl = _classes(rng, P)
    return dict(order=rng.permutation(P)[:n].astype(np.int32), hint=_hints(rng, P, N), cls=cls, ctrl=ctrl,
                ok=None if N == 0 or rng.random() < 0.5 else (rng.random(N) < 0.85).astype(np.uint8),
                li=int(rng.integers(0, 3 * N + 3)), brk=bool(rng.random() < 0.25))


def g_capacity(rng, enc, n_pods=None, bad=False):
    P, T, E, N = _sizes(enc)
    n = int(n_pods if n_pods is not None else rng.integers(0, min(P, 300) + 1))
    nreq = int(rng.integers(1, 6))
    off, pods = _split(rng, rng.permutation(P)[:n], nreq)
    kind = rng.integers(0, 2, nreq).astype(np.int32)
    if bad:
        kind[int(rng.integers(0, nreq))] = 7
    cls, ctrl = _classes(rng, P)
    return dict(kind=kind, off=off, pods=pods, hint=_hints(rng, P, N), cls=cls, ctrl=ctrl, li=int(rng.integers(0, 3 * N + 3)))


def g_removals(rng, enc, n_pods=None, persist=None):
    """candidates on distinct rows (row -1 holds no pods); the listed pending pods split over them"""
    P, T, E, N = _sizes(enc)
    rows = rng.permutation(N)[:int(rng.integers(0, min(N, 6) + 1))].tolist()
    if rng.random() < 0.3:
        rows.insert(int(rng.integers(0, len(rows) + 1)), -1)
    n = int(n_pods if n_pods is not None else rng.integers(0, min(P, 200) + 1))
    real = [i for i, r in enumerate(rows) if r >= 0]
    off, pods = _split(rng, rng.permutation(P)[:n] if real else [], max(len(real), 1))
    move_off, k = [0], 0
    for r in rows:
        if r >= 0 and k < len(real):
            move_off.append(int(off[k + 1]))
            k += 1
        else:
            move_off.append(move_off[-1])
    cls, ctrl = _classes(rng, P)
    return dict(cand=np.asarray(rows, np.int32), off=np.asarray(move_off, np.int32), pods=pods[:move_off[-1]],
                ok=None if N == 0 or rng.random() < 0.5 else (rng.random(N) < 0.9).astype(np.uint8),
                hint=_hints(rng, P, N), cls=cls, ctrl=ctrl, li=int(rng.integers(0, 3 * N + 3)),
                persist=bool(rng.random() < 0.5) if persist is None else persist)


def g_similar(rng, enc, bad=False):
    T = enc.T
    eligible = (rng.random(T) < 0.85).astype(np.uint8)
    if bad:
        eligible[int(rng.integers(0, T))] = 2
    max_size = rng.integers(0, 30, T).astype(np.int32)
    return dict(res_sig=rng.integers(0, 2, T).astype(np.int32),
                free_dims=(7 | rng.integers(0, 256, T) & rng.integers(0, 256, T)).astype(np.uint32),
                eligible=eligible, max_size=max_size, target_size=(rng.random(T) * (max_size + 3)).astype(np.int32),
                safe=_mask(rng, T, 0.9), ratios=tuple(float(x) for x in rng.choice([0.05, 0.015, 0.2], 3)))


def g_daemonsets(rng, enc, bad=False):
    T, S = enc.T, enc.struct.num_podspecs
    D = int(rng.choice([0, 1, 5, 33]))
    ds = rng.integers(0, S, D).astype(np.int32)
    if bad:
        ds = np.concatenate([ds, [S]]).astype(np.int32)
        D += 1
    run = None if D == 0 or rng.random() < 0.5 else rng.random((T, D)) < 0.2
    return dict(ds=ds, ev=_mask(rng, T, 0.8), run=run)


def g_eligibility(rng, enc, bad=False):
    N, nres = enc.struct.num_cluster_nodes, _n_res(enc)
    n = int(rng.integers(0, 2 * N + 1)) if N else 0
    cand = rng.integers(0, max(N, 1), n).astype(np.int32)
    if bad:
        cand = np.concatenate([cand, [N]]).astype(np.int32)
        n += 1
    flag = lambda p: None if rng.random() < 0.4 else (rng.random(n) < p).astype(np.uint8)
    return dict(cand=cand, gpu=rng.choice(np.array([-1, -1, -1, -2, 0, 1, 3], np.int32), n),
                thr=rng.choice(np.array([0.0, 0.3, 0.5, 0.9, 1.5]), n), skip_mirror=bool(rng.random() < 0.5),
                flags=None if rng.random() < 0.3 else rng.integers(0, 8, nres).astype(np.uint8),
                skip_ds=flag(0.5), pre=flag(0.1), unready=flag(0.1))


# ---- the runners: (engine, args) -> a tuple of arrays and numbers --------------------------------------------------------
def _vp(a):
    import ctypes
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def r_feasibility(e, a):
    enc = e.enc
    Pw = (enc.P + 31) // 32
    bits = np.zeros((enc.T, Pw), np.uint32) if a["bits"] else None
    reasons = np.zeros((enc.T, enc.P), np.uint8) if a["reasons"] else None
    count = np.zeros(enc.T, np.int32)
    e._check(e.lib.cae_feasibility(e.h, _vp(bits), _vp(reasons), _vp(count)))
    return bits, reasons, count


def r_feasibility_groups(e, a):
    return (e.feasibility_groups(),)


def r_group_reasons(e, a):
    return e.group_reasons(a["cons"], a["ex"], a["detail"])


def r_estimate(e, a):
    return e.estimate_all(a["caps"])


def r_estimate_ex(e, a):
    return e.estimate_all_li(a["caps"], a["li"])


def _price(e, a, rows):
    node_price, pod_price = _prices(e.enc)
    kw = dict(node_count=a["nc"], sched=a["sched"], order=a["order"]) if rows else {}
    return (e.price_scores(node_price, pod_price, a["stab"], a["cpu"], has_gpu=a["has_gpu"], exists=a["exists"], **kw),)


def r_price(e, a):
    return _price(e, a, False)


def r_price_rows(e, a):
    return _price(e, a, True)


def r_waste(e, a):
    return (e.waste_scores(),)


def r_expander(e, a):
    return e.expander_best(a["chain"], a["nc"], a["pc"], a.get("sched"))


def r_filter(e, a):
    return e.filter_schedulable(a["order"], a["hint"], a["cls"], a["ctrl"], a["ok"], a["li"], a["brk"])


def r_capacity(e, a):
    return e.check_capacity(a["kind"], a["off"], a["pods"], a["hint"], a["cls"], a["ctrl"], a["li"])


def r_removals(e, a):
    return e.simulate_removals(a["cand"], a["off"], a["pods"], a["ok"], a["hint"], a["cls"], a["ctrl"], a["li"], a["persist"])


def r_similar(e, a):
    return e.similar_node_groups(a["res_sig"], a["free_dims"], a["eligible"], a["max_size"], a["target_size"], (), a["safe"],
                                 a["ratios"])


def r_daemonsets(e, a):
    from kubernetes_autoscaler_b200.daemonset import pack_rows
    run = None if a["run"] is None else pack_rows(a["run"], len(a["ds"]))
    return e.template_daemonsets(a["ds"], a["ev"], run)


def r_eligibility(e, a):
    return e.scale_down_eligibility(a["cand"], a["gpu"], a["thr"], a["flags"], a["skip_ds"], a["skip_mirror"], a["pre"],
                                    a["unready"])


class Call:
    """kind: "plain" (answer = f(snapshot, args)), "estimate" (also becomes the last estimate), "consumer" (also reads the
    last estimate); `fn`: the C entry point; `bad`: a malformed variant (status -2)."""

    def __init__(self, fn, kind, gen, run, bad=False):
        self.fn, self.kind, self.gen, self.run, self.bad = fn, kind, gen, run, bad


def _bad(gen):
    return lambda rng, enc: gen(rng, enc, bad=True)


CATALOGUE = {
    "feasibility": Call("cae_feasibility", "plain", g_feasibility, r_feasibility),
    "feasibility_groups": Call("cae_feasibility_groups", "plain", g_none, r_feasibility_groups),
    "group_reasons": Call("cae_group_reasons", "plain", g_group_reasons, r_group_reasons),
    "estimate_all": Call("cae_estimate_all", "estimate", g_estimate, r_estimate),
    "estimate_all_ex": Call("cae_estimate_all_ex", "estimate", g_estimate_ex, r_estimate_ex),
    "waste_scores": Call("cae_waste_scores", "consumer", g_none, r_waste),
    "price_scores": Call("cae_price_scores", "consumer", g_price, r_price),
    "price_scores_rows": Call("cae_price_scores", "plain", g_price_rows, r_price_rows),
    "expander_best": Call("cae_expander_best", "consumer", g_expander, r_expander),
    "expander_best_rows": Call("cae_expander_best", "plain", g_expander_rows, r_expander),
    "filter_schedulable": Call("cae_filter_schedulable", "plain", g_filter, r_filter),
    "check_capacity": Call("cae_check_capacity", "plain", g_capacity, r_capacity),
    "simulate_removals": Call("cae_simulate_removals", "plain", g_removals, r_removals),
    "similar_node_groups": Call("cae_similar_node_groups", "plain", g_similar, r_similar),
    "template_daemonsets": Call("cae_template_daemonsets", "plain", g_daemonsets, r_daemonsets),
    "scale_down_eligibility": Call("cae_scale_down_eligibility", "plain", g_eligibility, r_eligibility),
    # malformed: status -2 before anything runs
    "group_reasons_bad": Call("cae_group_reasons", "plain", _bad(g_group_reasons), r_group_reasons, True),
    "estimate_all_ex_bad": Call("cae_estimate_all_ex", "plain", _bad(g_estimate_ex), r_estimate_ex, True),
    "check_capacity_bad": Call("cae_check_capacity", "plain", _bad(g_capacity), r_capacity, True),
    "similar_node_groups_bad": Call("cae_similar_node_groups", "plain", _bad(g_similar), r_similar, True),
    "template_daemonsets_bad": Call("cae_template_daemonsets", "plain", _bad(g_daemonsets), r_daemonsets, True),
    "scale_down_eligibility_bad": Call("cae_scale_down_eligibility", "plain", _bad(g_eligibility), r_eligibility, True),
}


def answer(eng, enc, name, args):
    """The call's answer on `eng` (holding `enc`): its outputs copied, or ("status", kind, message) when the engine refuses."""
    from kubernetes_autoscaler_b200.engine import EngineError
    eng.enc = enc
    try:
        out = CATALOGUE[name].run(eng, args)
    except EngineError as err:   # EngineUnsupported included: the status is part of the answer
        return ("status", type(err).__name__, str(err))
    return tuple(x.copy() if isinstance(x, np.ndarray) else x for x in out)


def refused(got):
    return isinstance(got[0], str) and got[0] == "status"


def check_status(name, got):
    """a malformed variant is refused with status -2; any other call is answered, or refused as a limit (status > 0)"""
    if CATALOGUE[name].bad:
        assert refused(got) and got[1] == "EngineError" and "status -2" in got[2], (name, got)
    else:
        assert not refused(got) or got[1] == "EngineUnsupported", (name, got)


def same(x, y):
    """bit for bit: doubles by their bits, arrays by dtype, shape and values"""
    if isinstance(x, tuple) or isinstance(y, tuple):
        return isinstance(x, tuple) and isinstance(y, tuple) and len(x) == len(y) and all(same(a, b) for a, b in zip(x, y))
    if isinstance(x, np.ndarray) or isinstance(y, np.ndarray):
        if not (isinstance(x, np.ndarray) and isinstance(y, np.ndarray)) or x.dtype != y.dtype or x.shape != y.shape:
            return False
        return same_bits(x, y) if x.dtype == np.float64 else bool(np.array_equal(x, y))
    return x == y


def args_key(args):
    return hashlib.sha1(pickle.dumps(sorted(args.items(), key=lambda kv: kv[0]))).hexdigest()


# ---- snapshots ------------------------------------------------------------------------------------------------------------
class Snap:
    """One loadable snapshot, identified by `sid` for the reference cache; `cluster` / `encoder`: the object world's cluster
    nodes and the encoder that interned them, where the snapshot was encoded from objects."""

    def __init__(self, sid, enc, cluster=None, encoder=None):
        self.sid, self.enc, self.cluster, self.encoder = sid, enc, cluster, encoder


def synth_snap(shape, seed=None):
    cfg, kw = SHAPES[shape]
    return Snap(("synth", shape, seed), synth.generate(cfg, **kw, **({} if seed is None else dict(seed=seed))))


def world_snap(seed, A=None, overfull=False, big=False):
    dims = None if A is None else rank_layout.DIM_SETS[A]
    cluster, templates, groups, namespaces, _ = fuzz._scenario(seed, big=big, dims=dims, overfull=overfull)
    encoder = Encoder()
    return Snap(("world", seed, A, overfull, big), encode(cluster, templates, groups, namespaces=namespaces, encoder=encoder),
                cluster, encoder)


def slab_snap(A, templates=4, seed=None, extra=64):
    """more pending pods than the estimator's shared window holds added nodes at A dims: an uncapped estimate takes the slab"""
    enc = synth.generate(1, pods=rank_layout.window_nodes(A) + extra, templates=templates, dims=rank_layout.DIM_SETS[A],
                         **({} if seed is None else dict(seed=seed)))
    return Snap(("slab", A, templates, seed, extra), enc)


def host_spread_snap(pods, seed=None):
    """C3 pods (hostname spread: the estimator's counter rows grow with the cap, dstride = domains + 1 + cap)"""
    return Snap(("c3", pods, seed), synth.generate(3, pods=pods, templates=12, cluster_nodes=24,
                                                    **({} if seed is None else dict(seed=seed))))


def has_host_counter(enc):
    return bool((np.asarray(enc.arrays["pts_key"]) == synth.K_HOST).any())


def reversed_groups(enc):
    """the same objects with the pending groups in reverse order: nodes, templates, pod specs, P and every counter's domains
    are those of `enc`, so the estimator's slab keeps its layout, while each group index names another spec"""
    go, ps = np.asarray(enc.arrays["group_off"]), np.asarray(enc.arrays["pend_spec"])
    parts = [ps[go[g]:go[g + 1]] for g in range(enc.E)][::-1]
    off = np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.int32)
    return enc.with_pending(np.concatenate(parts).astype(np.int32), off)


def twin(snap):
    return Snap(("reversed",) + tuple(snap.sid), reversed_groups(snap.enc))


# ---- the references -------------------------------------------------------------------------------------------------------
class Reference:
    """Single-call answers: a new engine loads the snapshot and makes only that call (a consumer: the sequence's last
    estimate with the same arguments, then the call).  Cached under (snapshot, call, arguments, last estimate).  The first
    time a (snapshot, call) is seen, the single-call engine also answers arguments drawn from a seed of (snapshot, call)
    alone, and that answer is checked against the oracle or a host mirror where the suite has one: which arguments are
    checked does not depend on which tests ran before."""

    def __init__(self, oracle=None):
        self.oracle = oracle
        self.cache = {}
        self.anchored = set()
        self.made = 0

    def want(self, snap, name, args, est=None):
        if self.oracle is not None and (snap.sid, name) not in self.anchored:
            self.anchored.add((snap.sid, name))
            rng = np.random.default_rng(zlib.crc32(repr((snap.sid, name)).encode()))
            fixed_est = ("estimate_all", g_estimate(rng, snap.enc)) if CATALOGUE[name].kind == "consumer" else None
            fixed = anchor_args(rng, snap, name)
            anchor(self.oracle, snap, name, fixed, fixed_est, self.single(snap, name, fixed, fixed_est))
        return self.single(snap, name, args, est)

    def single(self, snap, name, args, est):
        consumer = CATALOGUE[name].kind == "consumer"
        key = (snap.sid, name, args_key(args), (est[0], args_key(est[1])) if consumer else None)
        if key not in self.cache:
            from kubernetes_autoscaler_b200.engine import Engine
            e = Engine(device=0, want_reasons=True)
            self.made += 1
            try:
                e.load(snap.enc)
                if consumer:
                    assert not refused(answer(e, snap.enc, *est)), "the reference's estimate was refused"
                self.cache[key] = answer(e, snap.enc, name, args)
            finally:
                e.close()
        return self.cache[key]


ELIG_NOW = 1_700_000_000.0


def anchor_args(rng, snap, name):
    """the arguments a (snapshot, call) is anchored on.  Eligibility on an object world: pod flags from the resident pods
    themselves and GpuConfig resources by name, so that utilization_ref can restate the call on the objects."""
    args = CATALOGUE[name].gen(rng, snap.enc)
    if name == "scale_down_eligibility" and snap.cluster is not None:
        from kubernetes_autoscaler_b200.eligibility import cluster_pod_flags
        names = [None, None, "cpu", "memory", "nvidia.com/gpu", "example.com/none"]
        gpu = [names[i] for i in rng.integers(0, len(names), len(args["cand"]))]
        args.update(flags=cluster_pod_flags(snap.cluster, ELIG_NOW), gpu_names=gpu,
                    gpu=np.array([-1 if g is None else snap.encoder.resources.ids.get(g, -2) for g in gpu], np.int32))
    return args


def _oracle_estimate(oracle, enc, est):
    name, a = est
    if name == "estimate_all":
        return oracle.estimate_all(enc, a["caps"])[:4]
    return oracle.estimate_all_li(enc, a["caps"], a["li"])


def anchor(oracle, snap, name, a, est, got):
    """`got` (a single-call engine's answer) against the oracle, the DaemonSet mirror, the group-reason reference or the
    utilization restatement."""
    import group_reasons_ref
    import utilization_ref
    enc = snap.enc
    from kubernetes_autoscaler_b200.daemonset import run_bits_encoded, unpack_rows
    from kubernetes_autoscaler_b200.engine import unpack_bits
    check_status(name, got)
    if refused(got):
        return
    what = "%s against the oracle" % name
    if name == "feasibility":
        reasons, _ = oracle.feasibility_dense(enc)
        if a["bits"]:
            assert np.array_equal(unpack_bits(got[0], enc.P), reasons == 0), what
        if a["reasons"]:
            assert np.array_equal(got[1], reasons), what
        assert np.array_equal(got[2], (reasons == 0).sum(axis=1)), what
    elif name == "feasibility_groups":
        assert np.array_equal(got[0], oracle.feasibility_groups(enc)), what
    elif name == "group_reasons":
        sched, counts, detail = group_reasons_ref.group_reasons(enc, a["cons"], a["ex"])
        assert np.array_equal(got[0], sched) and np.array_equal(got[1], counts), what
        assert not a["detail"] or np.array_equal(got[2], detail), what
    elif name in ("estimate_all", "estimate_all_ex"):
        assert same(tuple(got), tuple(_oracle_estimate(oracle, enc, (name, a)))), what
    elif name in ("waste_scores", "expander_best", "price_scores"):
        nc, pc, sched, order = _oracle_estimate(oracle, enc, est)[:4]
        if name == "price_scores":
            node_price, pod_price = _prices(enc)
            want = oracle.price_scores(enc, node_price, pod_price, a["stab"], a["cpu"], has_gpu=a["has_gpu"], exists=a["exists"],
                                       node_count=nc, sched=sched, order=order)
            assert same_bits(got[0], want), what
        else:   # the scores come from the device-resident rows; the caller's counts only feed the chain
            assert same_bits(got[-1], oracle.expander(enc, CHAIN, nc, pc, sched)[1]), what
    elif name == "expander_best_rows":
        mask, waste = oracle.expander(enc, a["chain"], a["nc"], a["pc"], a["sched"])
        assert np.array_equal(got[0], mask) and same_bits(got[1], waste), what
    elif name == "price_scores_rows":
        node_price, pod_price = _prices(enc)
        want = oracle.price_scores(enc, node_price, pod_price, a["stab"], a["cpu"], has_gpu=a["has_gpu"], exists=a["exists"],
                                   node_count=a["nc"], sched=a["sched"], order=a["order"])
        assert same_bits(got[0], want), what
    elif name == "filter_schedulable":
        want = oracle.filter_schedulable(enc, a["order"], a["hint"], a["cls"], a["ctrl"], a["ok"], a["li"], a["brk"])
        assert np.array_equal(got[0], want[0]) and tuple(got[1:]) == tuple(want[1:]), what
    elif name == "template_daemonsets":
        want = run_bits_encoded(enc, a["ds"], a["ev"], a["run"])
        assert np.array_equal(unpack_rows(got[0], len(a["ds"])), want) and np.array_equal(got[1], want.sum(axis=1)), what
    elif name == "scale_down_eligibility" and snap.cluster is not None:
        st, util, reason, unneeded = utilization_ref.eligibility(snap.cluster, a["cand"], a["gpu_names"], a["thr"], ELIG_NOW,
                                                                 a["skip_ds"], a["skip_mirror"], a["pre"], a["unready"])
        assert st == 0 and same_bits(got[0], util), what
        assert np.array_equal(got[1], reason) and np.array_equal(got[2], unneeded), what
    # check_capacity, simulate_removals and similar_node_groups are checked against their host loops on object worlds in
    # their own files (ProvisioningRequests, drain lists, node-group sets); here their single-call engine is the reference


# ---- random sequences -----------------------------------------------------------------------------------------------------
PLAIN = sorted(n for n, c in CATALOGUE.items() if c.kind != "consumer")
CONSUMERS = sorted(n for n, c in CATALOGUE.items() if c.kind == "consumer")


def block_snaps(block):
    """The snapshots of one sequence block: synth shapes, object worlds (dynamic counters, hostname spread, overfull rows,
    a dim set), and one snapshot with more pending pods than the window holds nodes."""
    rnd = random.Random(0xC0DE + block)
    A = [2, 3, 5, 8, 0, 1, 4, 6, 7][block % 9]
    snaps = [synth_snap(["c2", "c3", "c4"][block % 3]), slab_snap(A)]
    for k in range(4):
        seed = 41_000 + 10 * block + k
        snaps.append(world_snap(seed, A=rnd.choice([None, 1, 3, 6]) if k == 1 else None, overfull=k == 2, big=k != 3))
    return snaps


def plan(seed, snaps, steps=None):
    """A sequence: [("load", i)] then 15-25 catalogue calls, now and then another load.  Consumers only after an estimate
    since the last load.  Returns [(op, snapshot index, args)]."""
    rng = np.random.default_rng(seed)
    n = int(steps if steps is not None else rng.integers(15, 26))
    cur = int(rng.integers(0, len(snaps)))
    out, estimated = [("load", cur, None)], False
    while len(out) < n + 1:
        if rng.random() < 0.1:
            cur = int(rng.integers(0, len(snaps)))
            out.append(("load", cur, None))
            estimated = False
            continue
        names = PLAIN + (CONSUMERS if estimated else [])
        name = names[int(rng.integers(0, len(names)))]
        out.append((name, cur, CATALOGUE[name].gen(rng, snaps[cur].enc)))
        estimated = estimated or CATALOGUE[name].kind == "estimate"
    return out
