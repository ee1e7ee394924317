#!/usr/bin/env python
"""The check-capacity ProvisioningRequest class on one engine, two ways, alternating in one process:

  batch   one cae_check_capacity over a booked request and K check requests;
  loop    the same on the ABI without it: per request cae_filter_schedulable(breakOnFailure), cae_force_add_pods for a
          found one (the pending indices, hints and classes remapped after it), then a cae_load to undo the placements.

    python scripts/check_capacity_tick.py --nodes 2000,15000 --k 10,100 --reps 5 [--check]

The cluster has --pods-per-node resident pods per node in 16 zones, a third of them under C3's zone spread; the requests
hold 8 to 1 000 pods of C3-like shapes (some spreading over zones), sized so that some are found and some are not.  Per
shape one JSON line: device_ms (CUDA events around the launch) and host_ms (wall time of the call) of the batch, host_ms
of the loop and its call count, the bytes each way uploaded, and whether both ways agree on every found flag, every pod's
node and lastIndex in every rep.  --check also runs the loop of single TrySchedulePods calls on the CPU oracle for the
first three requests and compares.  The card name and power limit are read in the same run."""
import argparse
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

HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


def world(n_nodes, pods_per_node, k, seed):
    from kubernetes_autoscaler_b200.objects import BuildTestNode, BuildTestPod, LabelSelector, NodeInfo, TopologySpreadConstraint, WithLabels
    from kubernetes_autoscaler_b200.provreq import PodSet, ProvisioningRequest
    rng = random.Random(seed)

    def shape(i, spread):
        p = BuildTestPod("s%d" % i, rng.choice([100, 250, 500, 1000, 2000]), rng.choice([256, 1024, 4096]) << 20,
                         WithLabels({"app": "a%d" % (i % 6)}))
        if spread:
            p.topology_spread = [TopologySpreadConstraint(rng.choice([1, 3]), ZONE, LabelSelector({"app": p.labels["app"]}))]
        return p
    shapes = [shape(i, i % 3 == 0) for i in range(24)]
    cluster = []
    for n in range(n_nodes):
        node = BuildTestNode("n%05d" % n, 16000, 64 << 30)
        node.labels = {HOST: node.name, ZONE: "z%d" % (n % 16)}
        node.allocatable["pods"] = node.capacity["pods"] = 110
        pods = []
        for j in range(pods_per_node):
            p = rng.choice(shapes).clone()
            p.name, p.node_name = "%s-%d" % (node.name, j), node.name
            p.owner_uid, p.owner_kind = "rs-" + p.labels["app"], "ReplicaSet"
            pods.append(p)
        cluster.append(NodeInfo(node, pods))
    reqs = []
    for r in range(k):
        n = rng.choice([8, 50, 200, 1000])
        sets = [PodSet(rng.choice(shapes), n // 2), PodSet(rng.choice(shapes), n - n // 2)]
        reqs.append(ProvisioningRequest("pr%d" % r, sets))
    # a quarter of the requests hold a pod larger than any node: not found whatever came before
    for r in reqs[::4]:
        r.pod_sets.append(PodSet(BuildTestPod("huge", 16001, 1), 1))
    booked = [ProvisioningRequest("booked", [PodSet(rng.choice(shapes), 200)])]
    return cluster, booked, reqs


def run_loop(eng, x, kinds, off, order, last_index):
    """The shim on the ABI without cae_check_capacity.  Returns (found per item, node per pod [P], lastIndex, calls, h2d)."""
    from kubernetes_autoscaler_b200.capi import CAE_CAPACITY_BOOK
    P = x.enc.P
    cur = x.enc
    idx = np.arange(P)                       # original pending index -> index in the engine now
    hint = x.hint if x.hint is not None else np.full(P, -1, np.int32)
    cls = x.sim_class
    assigned = np.full(P, -1, np.int32)
    found, calls, h2d = [], 0, 0
    for r, kind in enumerate(kinds):
        orig = np.asarray(order[off[r]:off[r + 1]])
        got, last_index, _ = eng.filter_schedulable(idx[orig], hint, cls, x.class_ctrl, None, last_index, kind != CAE_CAPACITY_BOOK)
        calls += 1
        h2d += eng.stats().h2d_bytes
        rows = got[idx[orig]]
        assigned[orig] = rows
        ok = bool((rows >= 0).all())
        found.append(ok)
        if (kind == CAE_CAPACITY_BOOK or ok) and (rows >= 0).any():
            moved = idx[orig][rows >= 0]
            after, new_index = cur.apply_force_add(moved, rows[rows >= 0])
            if eng.force_add_pods(moved, rows[rows >= 0], after) is False:
                eng.load(after)
            calls += 1
            h2d += eng.stats().h2d_bytes
            keep = new_index >= 0
            hint, cls = hint[keep], None if cls is None else cls[keep]
            idx = np.where(idx >= 0, new_index[np.maximum(idx, 0)], -1)
            cur = after
    eng.load(x.enc)                          # undo: the reference reverts its outer fork
    calls += 1
    h2d += eng.stats().h2d_bytes
    return found, assigned, last_index, calls, h2d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", default="2000,15000")
    ap.add_argument("--pods-per-node", type=int, default=30)
    ap.add_argument("--k", default="10,100")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import podlistprocessor as plp
    from kubernetes_autoscaler_b200.capi import CAE_CAPACITY_FOUND
    from kubernetes_autoscaler_b200.engine import Engine
    from kubernetes_autoscaler_b200.provreq import CapacityChecker
    eng = Engine(device=0)
    name, power = card()
    lines = []
    for n in [int(v) for v in a.nodes.split(",")]:
        for k in [int(v) for v in a.k.split(",")]:
            cluster, booked, reqs = world(n, a.pods_per_node, k, seed=n + k)
            items = CapacityChecker._items(booked, reqs)
            pods = [p for _, ps in items for p in ps]
            x = plp.prepare_try_schedule(cluster, pods)
            kinds = [kd for kd, _ in items]
            off = np.concatenate([[0], np.cumsum([len(ps) for _, ps in items])]).astype(np.int32)
            eng.load(x.enc)
            li0 = 12345
            dev, host, loop_host, agree, calls, loop_h2d, batch_h2d = [], [], [], True, 0, 0, 0
            for rep in range(a.reps + 1):
                t = time.perf_counter()
                res, assigned, li = eng.check_capacity(kinds, off, x.order, x.hint, x.sim_class, x.class_ctrl, li0)
                h = time.perf_counter() - t
                s = eng.stats()
                batch_h2d = s.h2d_bytes
                t = time.perf_counter()
                lfound, lassigned, lli, calls, loop_h2d = run_loop(eng, x, kinds, off, x.order, li0)
                lh = time.perf_counter() - t
                agree &= [r == CAE_CAPACITY_FOUND for r in res] == lfound and np.array_equal(assigned, lassigned) and li == lli
                if rep:   # the first rep warms up
                    dev.append(s.estimate_ms)
                    host.append(h * 1e3)
                    loop_host.append(lh * 1e3)
            line = dict(nodes=n, resident_pods=n * a.pods_per_node, k=k, pods=int(off[-1]), found=int(sum(r == CAE_CAPACITY_FOUND for r in res[1:])),
                        batch_device_ms=round(statistics.median(dev), 3), batch_host_ms=round(statistics.median(host), 3),
                        loop_host_ms=round(statistics.median(loop_host), 2), loop_calls=calls, batch_h2d_bytes=int(batch_h2d),
                        loop_h2d_bytes=int(loop_h2d), agree=bool(agree), device=name, power_limit=power)
            if a.check:
                sub = reqs[:3]
                o = CapacityChecker(cluster, schedulingSimulator=_oracle_sim())
                want = o.CheckCapacity(booked, sub)
                b = CapacityChecker(cluster, engine=eng)
                got = b.CheckCapacityBatch(booked, sub)
                line["oracle_agree"] = bool(want == got and o.assigned == b.assigned and
                                            o.schedulingSimulator.last_index == b.schedulingSimulator.last_index)
            print(json.dumps(line), flush=True)
            lines.append(line)
            assert agree, line
    if a.out:
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")
    eng.close()


def _oracle_sim():
    from capacity_harness import OracleSimulator
    return OracleSimulator()


if __name__ == "__main__":
    main()
