#!/usr/bin/env python
"""A scale-up tick after a change to the cluster, two ways, alternating in one process:

  delta tick   the delta call (below) + estimate_all + expander_best on an engine that holds the previous tick's snapshot;
  full tick    cae_load(the same new objects) + estimate_all + expander_best.

    python scripts/delta_tick.py --kind nodes --config 3 --scale 1,20,200,2000 --reps 5 [--check]
    python scripts/delta_tick.py --kind churn --config 3 --scale 1,10,100 --dirty 20 --reps 5 [--check]
    python scripts/delta_tick.py --kind pods --config 3 --scale 1,10,100 --reps 5 [--check]
    python scripts/delta_tick.py --kind placed --config 3 --reps 5 [--check]
    python scripts/delta_tick.py --kind templates --config 3 --scale 0,1,10,50 --reps 5 [--check]

Kinds, with the change `scale` stands for and the delta call:
  nodes  synth.node_churn on `scale` dirty nodes (binds, evictions, moves, cordons, taints, allocatable, relabels):
         cae_load_nodes(dirty rows) + cae_load_pending(pending rows);
  churn  synth.node_scale: `scale` nodes removed and `scale` added, plus synth.node_churn on --dirty rows:
         cae_load_node_churn(removed, added and dirty rows) + cae_load_pending(pending rows);
  pods   synth.pod_churn: `scale` new workloads arrive, `scale` pending groups finish: cae_load_pods(new specs + the new
         pending list).  The caller-side encode is not part of either tick (synth builds tables, not objects).
  templates  synth.template_churn: `scale` templates change, scale // 4 are removed and scale // 4 added (scale 0: a
         DaemonSet rollout, synth.daemonset_rollout, which changes every template's pod list): cae_load_templates.
  placed the reference's tick, filter pass then scale-up on ONE snapshot, three ways (`scale` is not used): every tick is
         cae_load + cae_filter_schedulable over all pending pods, then the placements become residents, then estimate_all +
         expander_best.  Tick A: cae_force_add_pods(what the pass assigned).  Tick B: the same placements as host-built
         deltas, cae_load_nodes(the complete new resident lists of the receiving rows) + cae_load_pods(the compacted
         pending list).  Tick C: a second cae_load of the objects after the placements.  Only the step that makes the
         placements resident is timed per tick, beside the tick; array work that builds B's deltas and C's objects is
         inside their ticks, since A needs none of it.
Also reported: the delta call's host wall time (cae_load_nodes and cae_load_node_churn return without a device
synchronise, cae_load_pods synchronises), its device time (CUDA events on the engine's stream) and the bytes it uploaded,
with the device name and power limit.  --check: both ticks' node counts, pod counts, sched, order and dense fit counts must
be identical in every rep."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

SCALES = {"nodes": "1,20,200,2000", "churn": "1,10,100", "pods": "1,10,100", "placed": "0", "templates": "0,1,10,50"}


def _card():
    import torch
    out = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        out["power_limit_w"], out["sm_max_mhz"] = float(q[0]), int(q[1])
    except Exception:
        out["power_limit_w"] = None
    return out


def _stats(xs):
    xs = sorted(xs)
    return {"median": float(np.median(xs)), "min": float(xs[0]), "max": float(xs[-1])}


def _change(synth, kind, enc, seed, scale, dirty):
    """The objects after the change, the delta call that applies it to an engine holding `enc` (True when it applied), and
    the pending-rows call that completes it (None: the delta call replaces the pending list itself)."""
    if kind == "nodes":
        delta, pending = synth.node_churn(enc, seed, scale)
        return pending.apply_node_delta(delta), lambda eng: eng.load_nodes(delta), lambda eng: eng.load_pending(pending)
    if kind == "churn":
        churn, pending = synth.node_scale(enc, seed, scale, scale, dirty)
        return pending.apply_node_churn(churn), lambda eng: eng.load_node_churn(churn), lambda eng: eng.load_pending(pending)
    if kind == "templates":
        delta = synth.template_churn(enc, seed, scale, scale // 4, scale // 4) if scale else synth.daemonset_rollout(enc, seed)
        after = enc.apply_template_delta(delta)
        return after, lambda eng: eng.load_templates(delta, after), None
    delta = synth.pod_churn(enc, seed, scale, scale)
    after = enc.apply_pod_delta(delta)
    return after, lambda eng: eng.load_pods(delta, after) == 0, None


def _placed_as_deltas(enc, pods, nodes):
    """The placements as the deltas a caller without cae_force_add_pods sends: the receiving rows as dirty rows with their
    unchanged node columns and complete new resident lists, and the pending list without the placed pods."""
    from kubernetes_autoscaler_b200.encode import NodeDelta, PodDelta
    after, _ = enc.apply_force_add(pods, nodes)
    a, b = enc.arrays, after.arrays
    rows = np.unique(nodes)
    off = b["node_pod_off"]
    lists = [b["node_pod_spec"][off[r]:off[r + 1]] for r in rows]
    nd = NodeDelta(row=rows, labelset=a["node_labelset"][rows], taint_list=a["node_taint_list"][rows],
                   unschedulable=a["node_unschedulable"][rows], alloc=a["node_alloc"][rows], allowed_pods=a["node_allowed_pods"][rows],
                   pod_off=np.concatenate([[0], np.cumsum([len(x) for x in lists])]), pod_spec=np.concatenate(lists))
    return after, nd, PodDelta(group_off=b["group_off"], pend_spec=b["pend_spec"])


def _placed(args):
    """--kind placed: ticks A, B and C of the module docstring, alternating, on three engines."""
    import __graft_entry__ as ge
    ge.build()
    import torch
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.engine import Engine
    enc = synth.generate(args.config, pods=args.pods, templates=args.templates, cluster_nodes=args.cluster_nodes)
    caps = np.full(enc.T, args.cap, np.int32)
    chain = [0, 1, 2]
    order = np.arange(enc.P, dtype=np.int32)[::-1].copy()
    engs = {k: Engine(device=0) for k in "ABC"}
    sa = torch.cuda.ExternalStream(engs["A"].stream(), device=torch.device("cuda", 0))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def tick(kind):
        eng = engs[kind]
        r = {}
        t0 = time.perf_counter()
        eng.load(enc)
        assigned, _, _ = eng.filter_schedulable(order)
        placed = np.ascontiguousarray(order[assigned[order] >= 0], np.int32)
        nodes = np.ascontiguousarray(assigned[placed], np.int32)
        t1 = time.perf_counter()
        if kind == "A":
            e0.record(sa)
            # the ABI call itself (the binding's force_add_pods also builds the new_index map in numpy)
            assert eng.lib.cae_force_add_pods(eng.h, len(placed), placed.ctypes.data, nodes.ctypes.data, None) == 0
            e1.record(sa)
            r["A_call_host_ms"] = 1e3 * (time.perf_counter() - t1)
            r["A_h2d_bytes"] = int(eng.stats().h2d_bytes)
        elif kind == "B":
            after, nd, pd = _placed_as_deltas(enc, placed, nodes)
            assert eng.load_nodes(nd)
            nbytes = int(eng.stats().h2d_bytes)
            assert eng.load_pods(pd, after) == 0
            r["B_h2d_bytes"] = nbytes + int(eng.stats().h2d_bytes)
        else:
            eng.load(enc.apply_force_add(placed, nodes)[0])
        t2 = time.perf_counter()
        nc, pc, sched, order_t = eng.estimate_all(caps, copy=False)
        eng.expander_best(chain, nc, pc)
        t3 = time.perf_counter()
        r["%s_tick_ms" % kind] = 1e3 * (t3 - t0)
        r["%s_placements_ms" % kind] = 1e3 * (t2 - t1)
        if kind == "A":
            e1.synchronize()
            r["A_call_dev_ms"] = e0.elapsed_time(e1)
            eng.enc = enc.apply_force_add(placed, nodes)[0]   # untimed: the binding's shapes (P changed) for the check below
        out = [x.copy() for x in (nc, pc, sched, order_t)] + [eng.feasibility(want_bits=False)[2].copy()] if args.check else None
        return r, out, len(placed)

    for k in "ABC":   # warm every shape the timed window uses
        tick(k)
    out = {"kind": "placed", "config": args.config, "pods": enc.P, "templates": enc.T,
           "cluster_nodes": enc.struct.num_cluster_nodes, "cap": args.cap, **_card()}
    rows, ok_all = [], True
    for rep in range(args.reps):
        r, outs = {}, {}
        for k in ("ABC", "BCA", "CAB")[rep % 3]:
            rk, outs[k], r["placed_pods"] = tick(k)
            r.update(rk)
        if args.check:
            r["same"] = all(np.array_equal(x, y) and np.array_equal(x, z) for x, y, z in zip(outs["A"], outs["B"], outs["C"]))
            ok_all &= r["same"]
        rows.append(r)
    run = {"reps": args.reps, "placed_pods": rows[0]["placed_pods"]}
    for k in rows[0]:
        if k not in ("same", "placed_pods"):
            run[k] = _stats([r[k] for r in rows])
    out["run"] = run
    out["check"] = ok_all if args.check else None
    print(json.dumps(out))
    for e in engs.values():
        e.close()
    if args.check and not ok_all:
        sys.exit(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", choices=sorted(SCALES), required=True)
    ap.add_argument("--config", type=int, choices=(3, 4), default=3)
    ap.add_argument("--scale", default=None, help="comma list of change sizes (default per kind: %s)" % SCALES)
    ap.add_argument("--dirty", type=int, default=20, help="dirty rows beside the removed and added nodes (churn)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cap", type=int, default=1000)
    ap.add_argument("--pods", type=int, default=None)
    ap.add_argument("--templates", type=int, default=None)
    ap.add_argument("--cluster-nodes", type=int, default=None)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    if args.kind == "placed":
        return _placed(args)
    import __graft_entry__ as ge
    ge.build()
    import torch
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.engine import Engine
    enc = synth.generate(args.config, pods=args.pods, templates=args.templates, cluster_nodes=args.cluster_nodes)
    caps = np.full(enc.T, args.cap, np.int32)
    chain = [0, 1, 2]
    a, b = Engine(device=0), Engine(device=0)
    sa = torch.cuda.ExternalStream(a.stream(), device=torch.device("cuda", 0))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for eng in (a, b):   # warm every shape the timed window uses
        eng.load(enc)
        nc, pc, _, _ = eng.estimate_all(caps, copy=False)
        eng.expander_best(chain, nc, pc)
    _, call, pend = _change(synth, args.kind, enc, 999, 8, 8)
    assert call(a) and (pend is None or pend(a))
    out = {"kind": args.kind, "config": args.config, "pods": enc.P, "templates": enc.T,
           "cluster_nodes": enc.struct.num_cluster_nodes, "cap": args.cap, **_card(), "runs": []}
    ok_all = True
    for scale in [int(x) for x in (args.scale or SCALES[args.kind]).split(",")]:
        rows = []
        for rep in range(args.reps):
            after, call, pend = _change(synth, args.kind, enc, 1000 * scale + rep, scale, args.dirty)
            a.load(enc)
            caps = np.full(after.T, args.cap, np.int32)   # a template delta changes T

            def delta_tick():
                t0 = time.perf_counter()
                e0.record(sa)
                assert call(a)
                e1.record(sa)
                t1 = time.perf_counter()
                nbytes = int(a.stats().h2d_bytes)
                assert pend is None or pend(a)
                nc, pc, sched, order = a.estimate_all(caps, copy=False)
                a.expander_best(chain, nc, pc)
                t2 = time.perf_counter()
                e1.synchronize()
                return {"delta_tick_ms": 1e3 * (t2 - t0), "delta_host_ms": 1e3 * (t1 - t0),
                        "delta_dev_ms": e0.elapsed_time(e1), "delta_h2d_bytes": nbytes}

            def full_tick():
                t0 = time.perf_counter()
                b.load(after)
                t1 = time.perf_counter()
                nc, pc, _, _ = b.estimate_all(caps, copy=False)
                b.expander_best(chain, nc, pc)
                t2 = time.perf_counter()
                return {"full_tick_ms": 1e3 * (t2 - t0), "full_load_ms": 1e3 * (t1 - t0)}

            r = {}
            for f in ((delta_tick, full_tick) if rep % 2 == 0 else (full_tick, delta_tick)):
                r.update(f())
            if args.check:
                got = [x.copy() for x in a.estimate_all(caps, copy=False)] + [a.feasibility(want_bits=False)[2].copy()]
                want = [x.copy() for x in b.estimate_all(caps, copy=False)] + [b.feasibility(want_bits=False)[2].copy()]
                r["same"] = all(np.array_equal(x, y) for x, y in zip(got, want))
                ok_all &= r["same"]
            rows.append(r)
        run = {"kind": args.kind, "scale": scale, "dirty": args.dirty if args.kind == "churn" else None, "reps": args.reps,
               "pending_after": after.P}
        for k in rows[0]:
            if k != "same":
                run[k] = _stats([r[k] for r in rows])
        run["speedup_median"] = run["full_tick_ms"]["median"] / run["delta_tick_ms"]["median"]
        if args.check:
            run["same"] = all(r["same"] for r in rows)
        out["runs"].append(run)
        print(json.dumps(run), flush=True)
    out["check"] = ok_all if args.check else None
    print(json.dumps(out))
    a.close()
    b.close()
    if args.check and not ok_all:
        sys.exit(1)


if __name__ == "__main__":
    main()
