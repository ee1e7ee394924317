#!/usr/bin/env python
"""A scale-up tick after a change to the cluster, two ways, alternating in one process:

  delta tick   the delta call (below) + estimate_all + expander_best on an engine that holds the previous tick's snapshot;
  full tick    cae_load(the same new objects) + estimate_all + expander_best.

    python scripts/delta_tick.py --kind nodes --config 3 --scale 1,20,200,2000 --reps 5 [--check]
    python scripts/delta_tick.py --kind churn --config 3 --scale 1,10,100 --dirty 20 --reps 5 [--check]
    python scripts/delta_tick.py --kind pods --config 3 --scale 1,10,100 --reps 5 [--check]

Kinds, with the change `scale` stands for and the delta call:
  nodes  synth.node_churn on `scale` dirty nodes (binds, evictions, moves, cordons, taints, allocatable, relabels):
         cae_load_nodes(dirty rows) + cae_load_pending(pending rows);
  churn  synth.node_scale: `scale` nodes removed and `scale` added, plus synth.node_churn on --dirty rows:
         cae_load_node_churn(removed, added and dirty rows) + cae_load_pending(pending rows);
  pods   synth.pod_churn: `scale` new workloads arrive, `scale` pending groups finish: cae_load_pods(new specs + the new
         pending list).  The caller-side encode is not part of either tick (synth builds tables, not objects).
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

SCALES = {"nodes": "1,20,200,2000", "churn": "1,10,100", "pods": "1,10,100"}


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
    delta = synth.pod_churn(enc, seed, scale, scale)
    after = enc.apply_pod_delta(delta)
    return after, lambda eng: eng.load_pods(delta, after) == 0, None


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
