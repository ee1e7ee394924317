#!/usr/bin/env python
"""cae_scale_down_eligibility on a cluster of --nodes nodes with --pods resident pods each (default 2 000 x 30, the cluster
size of C3, and 15 000 x 30), every node a candidate.  Per size, one JSON line:

  * device_ms: CUDA events on the engine's stream around the call (median of --reps after a warm-up): the H2D copy of the
    inputs (the pod flags are most of it), both kernels and the D2H copy of the outputs;
  * host_ms: host wall time of the call (it ends in a stream synchronise), median; checker_ms: Checker.FilterOutUnremovable
    end to end, which also builds the pod flags and the per-candidate vectors in Python, median;
  * python_ref_ms: the CPU restatement (tests/utilization_ref.py) over every candidate, once.  It is Python: the cost of the
    Go loop it stands for (utilization.Calculate per candidate) is not measured;
  * tick_ms: the composed tick on the scale-up load, Checker.FilterOutUnremovable then RemovalSimulator.SimulateNodeRemovals
    on the first --removals unneeded nodes (prepare, removal load and cae_simulate_removals), once after a warm-up;
  * resident_tick_ms: the same tick with RemovalSimulator.SimulateNodeRemovalsResident on the same engine, without the
    removal load (slots, cae_simulate_resident_removals), once after a warm-up; resident_call_ms: CUDA events on the
    engine's stream around that call (the slot upload, the spec gather, the movers' derivation, the batch and its log).
    Both ticks must give the same outcome.
The engine's answers are checked against the restatement.  The card name and power limit are read in the same run."""
import argparse
import copy
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402

from similar_groups_tick import card  # noqa: E402

NOW = 1_700_000_000.0


def world(n_nodes, pods_per_node, seed):
    """n_nodes nodes of 16 cores / 64 GiB, each with pods_per_node pods drawn from a pool of plain, DaemonSet, mirror and
    long-terminating pods whose requests put the nodes on both sides of a 0.5 threshold"""
    from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, NodeInfo
    rng = random.Random(seed)
    pool = []
    for i in range(64):
        p = BuildTestPod("p%d" % i, rng.choice([50, 100, 250, 500, 1000]), rng.choice([64, 256, 1024, 2048]) << 20)
        if i % 8 == 1:
            p.owner_kind, p.owner_uid = "DaemonSet", "ds%d" % i
        elif i % 16 == 2:
            p.annotations = {"kubernetes.io/config.mirror": "x"}
        elif i % 32 == 3:
            p.terminating, p.deletion_timestamp = True, NOW - 3600
        else:
            p.owner_kind, p.owner_uid = "ReplicaSet", "rs%d" % i
        pool.append(p)
    cluster = []
    for n in range(n_nodes):
        node = BuildTestNode("n%d" % n, 16000, 64 << 30)
        node.labels = {"kubernetes.io/hostname": node.name}
        node.allocatable["pods"] = node.capacity["pods"] = 110
        pods = []
        for j in range(pods_per_node):             # one object per pod: the removal batch tells pods apart by name
            p = copy.copy(rng.choice(pool))
            p.name = "%s-%d" % (node.name, j)
            pods.append(p)
        cluster.append(NodeInfo(node, pods))
    return cluster


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", default="2000,15000")
    ap.add_argument("--pods", type=int, default=30)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--removals", type=int, default=200)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    import utilization_ref as ref
    from kubernetes_autoscaler_b200.eligibility import Checker, NodeGroupConfig, cluster_pod_flags
    from kubernetes_autoscaler_b200.encode import Encoder, encode
    from kubernetes_autoscaler_b200.engine import Engine
    from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, NodeInfo, makePodEquivalenceGroup
    from kubernetes_autoscaler_b200.removal import RemovalSimulator
    name, power = card()
    eng = Engine(device=0)
    stream = torch.cuda.ExternalStream(eng.stream())
    out = open(a.out, "w") if a.out else None
    for N in [int(x) for x in a.nodes.split(",")]:
        cluster = world(N, a.pods, N)
        encoder = Encoder()
        enc = encode(cluster, [NodeInfo(BuildTestNode("t", 16000, 64 << 30))], [makePodEquivalenceGroup(BuildTestPod("x", 1, 1), 1)],
                     encoder=encoder)
        eng.load(enc)
        names = [ni.node.name for ni in cluster]
        rows = np.arange(N, dtype=np.int32)
        gdim = np.full(N, -1, np.int32)
        th = np.full(N, 0.5)
        skip_ds = (rows % 2).astype(np.uint8)
        flags = cluster_pod_flags(cluster, NOW)

        def timed():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            t0 = time.perf_counter()
            r = eng.scale_down_eligibility(rows, gdim, th, flags, skip_ds, True)
            t1 = time.perf_counter()
            e1.record(stream)
            e1.synchronize()
            return r, e0.elapsed_time(e1), (t1 - t0) * 1e3
        (util, reason, unneeded), _, _ = timed()
        t0 = time.perf_counter()
        st, wutil, wreason, wunneeded = ref.eligibility(cluster, rows, [None] * N, th, NOW, skip_ds, True)
        python_ms = (time.perf_counter() - t0) * 1e3
        assert st == 0 and ref.same_bits(util, wutil) and np.array_equal(reason, wreason) and np.array_equal(unneeded, wunneeded)
        dev, host = [], []
        for _ in range(a.reps):
            r, d, hms = timed()
            assert np.array_equal(r[2], unneeded)
            dev.append(d)
            host.append(hms)
        h2d = int(eng.stats().h2d_bytes)
        groups = {nm: NodeGroupConfig(0.5, 0.5, bool(i % 2)) for i, nm in enumerate(names)}
        checker = Checker(eng, encoder.resources.ids, ignore_mirror_pods_utilization=True)
        chk = []
        for _ in range(max(a.reps // 4, 3)):
            t0 = time.perf_counter()
            un, umap, inel = checker.FilterOutUnremovable(cluster, names, NOW, groups)
            chk.append((time.perf_counter() - t0) * 1e3)
        assert un == [names[i] for i in unneeded]
        dest = {nm: True for nm in names}

        def tick():
            eng.load(enc)                                  # the tick's scale-up load, which the checker reads
            t0 = time.perf_counter()
            un, _, _ = checker.FilterOutUnremovable(cluster, names, NOW, groups)
            res = RemovalSimulator(cluster, engine=eng).SimulateNodeRemovals(un[:a.removals], dest)
            return (time.perf_counter() - t0) * 1e3, res
        tick()
        tick_ms, res = tick()
        call_ms = []
        call = eng.simulate_resident_removals

        def timed_call(*args, **kw):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            r = call(*args, **kw)
            e1.record(stream)
            e1.synchronize()
            call_ms.append(e0.elapsed_time(e1))
            return r
        eng.simulate_resident_removals = timed_call

        def resident_tick():
            eng.load(enc)
            t0 = time.perf_counter()
            un, _, _ = checker.FilterOutUnremovable(cluster, names, NOW, groups)
            res = RemovalSimulator(cluster, engine=eng).SimulateNodeRemovalsResident(un[:a.removals], dest)
            return (time.perf_counter() - t0) * 1e3, res
        resident_tick()
        resident_ms, res2 = resident_tick()
        del eng.simulate_resident_removals

        def outcome(rs):
            return [(r.node.name, [p.name for p in r.pods_to_reschedule], [p.name for p in r.daemonset_pods]) if r is not None
                    else (u.node.name, u.reason) for r, u in rs]
        assert outcome(res2) == outcome(res), "the resident tick differs from the tick with a removal load"
        row = dict(nodes=N, pods_per_node=a.pods, card=name, power_limit=power, candidates=N, unneeded=len(unneeded),
                   device_ms=round(statistics.median(dev), 4), host_ms=round(statistics.median(host), 4),
                   checker_ms=round(statistics.median(chk), 2), python_ref_ms=round(python_ms, 1),
                   h2d_bytes=h2d, tick_ms=round(tick_ms, 1), tick_removals=min(a.removals, len(unneeded)),
                   tick_removable=sum(r[0] is not None for r in res), resident_tick_ms=round(resident_ms, 1),
                   resident_call_ms=round(call_ms[-1], 3))
        line = json.dumps(row)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
