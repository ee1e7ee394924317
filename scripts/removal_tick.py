#!/usr/bin/env python
"""A scale-down tick: K node-removal simulations with persistence on, two ways, alternating in one process on one engine:

  per-candidate   RemovalSimulator.SimulateNodeRemoval in a loop (one encode, one cae_load and one
                  cae_filter_schedulable per candidate);
  batch           RemovalSimulator.SimulateNodeRemovals: one encode (prepare_removals), one cae_load and one
                  cae_simulate_removals, each timed on its own.

    python scripts/removal_tick.py --nodes 2000 --pods-per-node 30 --k 10,50,200 --reps 3

The cluster is object-level: nodes in zones with hostname labels, ~pods-per-node resident ReplicaSet pods each (some
under zone or hostname spread, some with hostname anti-affinity), a DaemonSet pod per node.  Every rep checks that both
ways give identical results, pods_to_reschedule, hints, lastIndex and final cluster.  Prints one JSON line per K with the
device name and power limit."""
import argparse
import copy
import json
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


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


def cluster(nodes, ppn, seed=0):
    from kubernetes_autoscaler_b200.objects import (BuildTestNode, BuildTestPod, LabelSelector, NodeInfo, PodAffinityTerm,
                                                    TopologySpreadConstraint, WithLabels)
    rng = random.Random(seed)
    out = []
    for i in range(nodes):
        n = BuildTestNode("node-%04d" % i, 32000, 128 << 30)
        n.labels = {HOST: n.name, ZONE: "zone-%d" % (i % 3)}
        pods = []
        for j in range(rng.randint(ppn // 2, ppn + ppn // 2)):
            app = "app-%d" % rng.randrange(40)
            p = BuildTestPod("p-%04d-%02d" % (i, j), rng.choice([100, 250, 500, 1000]), rng.choice([256, 512, 1024]) << 20,
                             WithLabels({"app": app}))
            p.owner_uid, p.owner_kind = "rs-" + app, "ReplicaSet"
            r = rng.random()
            if r < 0.15:
                p.topology_spread = [TopologySpreadConstraint(2, ZONE, LabelSelector({"app": app}))]
            elif r < 0.2:
                p.topology_spread = [TopologySpreadConstraint(3, HOST, LabelSelector({"app": app}))]
            elif r < 0.25:
                p.pod_anti_affinity = [PodAffinityTerm(LabelSelector({"app": app}), HOST)]
            pods.append(p)
        ds = BuildTestPod("ds-%04d" % i, 50, 64 << 20)
        ds.owner_uid, ds.owner_kind = "ds", "DaemonSet"
        out.append(NodeInfo(n, pods + [ds]))
    return out


def outcome(results, sim, cl):
    res = [("remove", a.node.name, [p.name for p in a.pods_to_reschedule]) if a is not None else ("keep", b.node.name, b.reason)
           for a, b in results]
    return res, dict(sim.hints.current), sim.last_index, [(ni.node.name, [p.name for p in ni.pods]) for ni in cl]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=2000)
    ap.add_argument("--pods-per-node", type=int, default=30)
    ap.add_argument("--k", default="10,50,200")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    from kubernetes_autoscaler_b200.engine import Engine
    from kubernetes_autoscaler_b200.removal import RemovalSimulator
    eng = Engine(device=0)
    base = cluster(a.nodes, a.pods_per_node)
    card = _card()
    rng = random.Random(1)
    for k in [int(v) for v in a.k.split(",")]:
        cands = rng.sample([ni.node.name for ni in base], k)
        dest = {ni.node.name: True for ni in base}
        loop_s, enc_s, load_s, call_s, batch_s = [], [], [], [], []
        same = True
        for rep in range(a.reps + 1):   # rep 0 warms up
            for way in ("loop", "batch") if rep % 2 == 0 else ("batch", "loop"):
                cl = copy.deepcopy(base)
                sim = plp.HintingSimulator(eng)
                r = RemovalSimulator(cl, True, schedulingSimulator=sim)
                if way == "loop":
                    t0 = time.perf_counter()
                    res = [r.SimulateNodeRemoval(n, dest) for n in cands]
                    dt = time.perf_counter() - t0
                    if rep:
                        loop_s.append(dt)
                    want = outcome(res, sim, cl)
                else:
                    t0 = time.perf_counter()
                    x = plp.prepare_removals(cl, cands, dest, None, sim.hints)
                    t1 = time.perf_counter()
                    eng.load(x.enc)
                    t2 = time.perf_counter()
                    out = eng.simulate_removals(x.cand_node, x.move_off, x.move_pod, x.dest_ok, x.hint, x.sim_class, x.class_ctrl,
                                                sim.last_index, True)
                    t3 = time.perf_counter()
                    res = r._apply_removals(x, *out)
                    t4 = time.perf_counter()
                    if rep:
                        enc_s.append(t1 - t0); load_s.append(t2 - t1); call_s.append(t3 - t2); batch_s.append(t4 - t0)
                    got = outcome(res, sim, cl)
            same = same and got == want
        print(json.dumps(dict(card, nodes=a.nodes, pods=sum(len(ni.pods) for ni in base), k=k, persist=True, reps=a.reps,
                              removable=sum(1 for v in want[0] if v[0] == "remove"), identical=same,
                              per_candidate_s=_stats(loop_s), batch_s=_stats(batch_s), batch_encode_s=_stats(enc_s),
                              batch_load_s=_stats(load_s), batch_call_s=_stats(call_s))), flush=True)
        if not same:
            sys.exit("batch and per-candidate results differ at K=%d" % k)
    eng.close()


if __name__ == "__main__":
    main()
