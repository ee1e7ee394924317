#!/usr/bin/env python
"""One autoscaler loop with a scale-up's upcoming nodes in the snapshot, three ways, alternating in one process:

  A  cae_add_upcoming_nodes(the copies) on an engine holding the loop's snapshot without them;
  B  cae_load_node_churn with the copies built on the host as added rows (each copy's columns and template pod list read
     from the objects, inside the loop) on an engine holding the same snapshot;
  C  cae_load of the objects with the copies (EncodedObjects.apply_upcoming inside the loop).

    python scripts/upcoming_tick.py --config 3,4 --upcoming 10,100,1000 --reps 5 [--check]

Each loop then runs what follows in RunOnce: the filter-out-schedulable pass over every pending pod, cae_force_add_pods of
its placements, estimate_all and expander_best.  The copies are `upcoming` nodes spread round-robin over the templates,
each with its template's labels and a new hostname value.  Reported per (config, upcoming): the loop's wall time per way,
the upcoming call's host wall time (it returns without a device synchronise), its device time (CUDA events on the
engine's stream) and the bytes it uploaded, the same for B's churn call, and the card name and power limit read in the
same run.  --check: the filter pass's assignments, the estimate's node counts, pod counts, sched and order, and the
expander's choice must be identical across the three ways in every rep (exit 1 otherwise)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from delta_tick import _card, _stats  # noqa: E402


def _upcoming(enc, k):
    """UpcomingNodes of k copies (template j % T for copy j) against `enc`, with their label sets as tails"""
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.encode import NodeChurn, NodeDelta, UpcomingNodes
    a, s = enc.arrays, enc.struct
    N, T = s.num_cluster_nodes, enc.T
    tmpl = [j % T for j in range(k)]
    pairs = []
    for j, t in enumerate(tmpl):
        ls = int(a["node_labelset"][N + t])
        lab = dict(zip(a["ls_key"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist(), a["ls_val"][a["ls_off"][ls]:a["ls_off"][ls + 1]].tolist()))
        lab[synth.K_HOST] = s.num_values + j
        pairs.append(sorted(lab.items()))
    tails = NodeDelta(value_is_int=np.zeros(k), value_int=np.zeros(k),
                      ls_off=np.concatenate([[0], np.cumsum([len(p) for p in pairs])]),
                      ls_key=[x for p in pairs for x, _ in p], ls_val=[v for p in pairs for _, v in p])
    name0 = int(a["node_name"].max(initial=0)) + 1
    return UpcomingNodes(NodeChurn(tails), template_idx=tmpl, name=np.arange(name0, name0 + k),
                         labelset=s.num_labelsets + np.arange(k))


def _as_churn(enc, up):
    """The same copies as the added rows of a cae_load_node_churn: the host reads each copy's columns and pod list"""
    from kubernetes_autoscaler_b200.encode import NodeChurn
    a, N = enc.arrays, enc.struct.num_cluster_nodes
    tr = N + up.arrays["template_idx"].astype(np.int64)
    off, spec = a["node_pod_off"], a["node_pod_spec"]
    cnt = off[tr + 1] - off[tr]
    pod_spec = np.concatenate([spec[off[r]:off[r + 1]] for r in tr]) if len(tr) else []
    return NodeChurn(up.churn.changed, name=up.arrays["name"], labelset=up.arrays["labelset"], taint_list=a["node_taint_list"][tr],
                     unschedulable=a["node_unschedulable"][tr], alloc=a["node_alloc"][tr], allowed_pods=a["node_allowed_pods"][tr],
                     pod_off=np.concatenate([[0], np.cumsum(cnt)]), pod_spec=pod_spec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="3,4")
    ap.add_argument("--upcoming", default="10,100,1000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cap", type=int, default=1000)
    ap.add_argument("--pods", type=int, default=None)
    ap.add_argument("--templates", type=int, default=None)
    ap.add_argument("--cluster-nodes", type=int, default=None)
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.engine import Engine
    engs = {k: Engine(device=0) for k in "ABC"}
    ev = {k: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for k in "AB"}
    streams = {k: torch.cuda.ExternalStream(engs[k].stream(), device=torch.device("cuda", 0)) for k in "AB"}
    chain = [0, 1, 2]
    ok_all = True
    for config in [int(x) for x in args.config.split(",")]:
        enc = synth.generate(config, pods=args.pods, templates=args.templates, cluster_nodes=args.cluster_nodes)
        caps = np.full(enc.T, args.cap, np.int32)
        head = {"config": config, "pods": enc.P, "templates": enc.T, "cluster_nodes": enc.struct.num_cluster_nodes,
                "cap": args.cap, **_card()}

        def loop(kind, up, shapes):
            """`shapes`: the objects after the copies, stated beforehand for the binding of A and B (C states them itself,
            as the caller's encode of a full load)"""
            eng = engs[kind]
            eng.load(enc)          # the loop's snapshot without the copies (untimed)
            r = {}
            t0 = time.perf_counter()
            if kind == "C":
                after = enc.apply_upcoming(up)
                eng.load(after)
            else:
                e0, e1 = ev[kind]
                churn = _as_churn(enc, up) if kind == "B" else None
                t1 = time.perf_counter()
                e0.record(streams[kind])
                assert eng.add_upcoming_nodes(up) if kind == "A" else eng.load_node_churn(churn)
                e1.record(streams[kind])
                r[kind + "_call_host_ms"] = 1e3 * (time.perf_counter() - t1)
                r[kind + "_h2d_bytes"] = int(eng.stats().h2d_bytes)
                after = eng.enc = shapes
            order = np.arange(after.P, dtype=np.int32)
            assigned, li, _ = eng.filter_schedulable(order)
            placed = np.flatnonzero(assigned[:after.P] >= 0).astype(np.int32)
            nodes = np.ascontiguousarray(assigned[placed], np.int32)
            if len(placed):
                assert eng.lib.cae_force_add_pods(eng.h, len(placed), placed.ctypes.data, nodes.ctypes.data, None) == 0
            nc, pc, sched, order_t = eng.estimate_all(caps, copy=False)
            best = eng.expander_best(chain, nc, pc)
            torch.cuda.synchronize()
            r[kind + "_loop_ms"] = 1e3 * (time.perf_counter() - t0)
            if kind != "C":
                e1.synchronize()
                r[kind + "_call_dev_ms"] = e0.elapsed_time(e1)
            out = [assigned[:after.P].copy(), np.int64(li), nc.copy(), pc.copy(), sched.copy(), order_t.copy(),
                   np.asarray(best[0]).copy()] if args.check else None
            return r, out, len(placed)

        warm = _upcoming(enc, 4)
        for k in "ABC":   # warm every shape the timed window uses
            loop(k, warm, enc.apply_upcoming(warm))
        for k in [int(x) for x in args.upcoming.split(",")]:
            up = _upcoming(enc, k)
            shapes = enc.apply_upcoming(up)
            rows = []
            for rep in range(args.reps):
                r, outs = {}, {}
                for kind in ("ABC", "BCA", "CAB")[rep % 3]:
                    rk, outs[kind], r["placed_pods"] = loop(kind, up, shapes)
                    r.update(rk)
                if args.check:
                    r["same"] = all(np.array_equal(x, y) and np.array_equal(x, z) for x, y, z in zip(outs["A"], outs["B"], outs["C"]))
                    ok_all &= r["same"]
                rows.append(r)
            run = {"upcoming": k, "reps": args.reps, "placed_pods": rows[0]["placed_pods"]}
            for key in rows[0]:
                if key not in ("same", "placed_pods"):
                    run[key] = _stats([r[key] for r in rows])
            run["check"] = all(r["same"] for r in rows) if args.check else None
            print(json.dumps({**head, **run}), flush=True)
    for e in engs.values():
        e.close()
    if args.check and not ok_all:
        sys.exit(1)


if __name__ == "__main__":
    main()
