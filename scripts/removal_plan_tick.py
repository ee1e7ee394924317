#!/usr/bin/env python
"""cae_plan_removals on the synthetic snapshot of scale_down_tick.py: --nodes nodes (default 2 000 and 15 000) with --pods
resident pods each, the first --cands unneeded candidates of cae_scale_down_eligibility, and --pdbs PDBs (default 0, 200
and 2 000).  Half of the PDBs select every pod of the namespace (DoesNotExist on a key no pod has), half select none, with
budgets no candidate exhausts, so every candidate is simulated and every mover counts against B/2 budgets.  One JSON line
per (nodes, B):

  * call_ms: CUDA events on the engine's stream recorded right before and after the C call cae_plan_removals alone (median
    of --reps after a warm-up), so the binding's Python is outside the window: the staged upload, the PDB match with its
    sync for the list size, the drain scan, the batch, the read-back and the host work between them inside the call;
  * batch_ms: the removal batch kernel alone (the engine's events around launch_removals, cae_stats.estimate_ms);
  * match_ms: the device time of pdb_match_kernel alone (both passes), from torch.profiler in a run of its own;
  * host_ms: host wall time of Engine.plan_removals (the binding's listing of the potential movers included), median;
  * h2d_bytes, d2h_bytes: cae_stats of the last call;
  * at B = 0, resident_call_ms / resident_batch_ms: the same two numbers for cae_simulate_resident_removals on the same
    movers, persisted, alternating with the plan call: the difference is the planner logic's cost.
--check compares the engine with the host loop on the CPU oracle (planner.categorize_nodes) at a small size first.  The card
name and power limit are read in the same run."""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
import numpy as np  # noqa: E402

from scale_down_tick import NOW, world  # noqa: E402
from similar_groups_tick import card  # noqa: E402


def pdbs_for(B):
    from kubernetes_autoscaler_b200.objects import LabelSelector, PodDisruptionBudget, Requirement
    return [PodDisruptionBudget("pdb%d" % b, "default",
                                LabelSelector(match_expressions=[Requirement("k%d" % (b % 50), "DoesNotExist" if b % 2 == 0 else "Exists")]),
                                10 ** 6) for b in range(B)]


def check(eng):
    import copy
    import plan_harness as ph
    rng = random.Random(3)
    cluster = world(60, 10, 60)
    for ni in cluster:
        for p in ni.pods:
            p.labels = {"app": rng.choice(["a", "b", "c"])}
    by = ph.random_bytes(rng, cluster)
    pdbs = ph.random_pdbs(rng, cluster, 40)
    cands = [ni.node.name for ni in cluster[:20]]
    for persist in (False, True):
        got = ph.engine_plan(eng, copy.deepcopy(cluster), cands, ph.everywhere(cluster), persist, by, pdbs, limit=12)
        want = ph.loop_plan(copy.deepcopy(cluster), cands, ph.everywhere(cluster), persist, by, pdbs, limit=12)
        assert got == want, "the engine differs from the host loop"
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", default="2000,15000")
    ap.add_argument("--pods", type=int, default=30)
    ap.add_argument("--cands", type=int, default=200)
    ap.add_argument("--pdbs", default="0,200,2000")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import drain as dr
    from kubernetes_autoscaler_b200.encode import Encoder, RemovalPlan, encode
    from kubernetes_autoscaler_b200.engine import Engine
    from kubernetes_autoscaler_b200.planner import encode_pdbs
    name, power = card()
    eng = Engine(device=0)
    checked = check(eng) if a.check else None
    stream = torch.cuda.ExternalStream(eng.stream())
    out = open(a.out, "w") if a.out else None

    call_ms = {}

    def around_c_call(name):
        """Replace the library's entry point `name` by one that records CUDA events right around the C call."""
        raw = getattr(eng.lib, name)

        def wrapped(*args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            rc = raw(*args)
            e1.record(stream)
            e1.synchronize()
            call_ms[name] = e0.elapsed_time(e1)
            return rc
        setattr(eng.lib, name, wrapped)
    around_c_call("cae_plan_removals")
    around_c_call("cae_simulate_resident_removals")

    def timed(fn, name):
        t0 = time.perf_counter()
        r = fn()
        host = (time.perf_counter() - t0) * 1e3
        return r, call_ms[name], float(eng.stats().estimate_ms), host

    for N in [int(x) for x in a.nodes.split(",")]:
        cluster = world(N, a.pods, N)
        encoder = Encoder()
        enc = encode(cluster, [], [], encoder=encoder)
        eng.load(enc)
        rows = np.arange(N, dtype=np.int32)
        flags = np.concatenate([[1 if p.owner_kind == "DaemonSet" else 0 for p in ni.pods] for ni in cluster]).astype(np.uint8)
        _, _, unneeded = eng.scale_down_eligibility(rows, np.full(N, -1, np.int32), np.full(N, 0.5), flags)
        cand = np.ascontiguousarray(unneeded[:a.cands], np.int32)
        drain = np.array([dr.drain_byte(p, NOW) for ni in cluster for p in ni.pods], np.uint8)
        for B in [int(x) for x in a.pdbs.split(",")]:
            eng.load(enc)
            plan = RemovalPlan(cand_node=cand, drain=drain, unneeded_limit=-1, kube_system_ns=-1, persist=1,
                               **encode_pdbs(encoder, eng.enc.struct.num_values, pdbs_for(B)))
            first = eng.plan_removals(plan)
            after = eng.enc                      # the objects every later call leaves: not restated in the timed window
            dev, batch, host = [], [], []
            res_dev, res_batch = [], []
            if B == 0:   # the resident batch on the same movers, alternating
                mo, ms = first["move_off"], first["move_slot"]
                eng.simulate_resident_removals(cand, mo, ms, persist=True, enc=after)
            for _ in range(a.reps):
                r, d, b, h = timed(lambda: eng.plan_removals(plan, enc=after), "cae_plan_removals")
                assert np.array_equal(r["result"], first["result"]) and np.array_equal(r["log"], first["log"])
                st = eng.stats()
                dev.append(d)
                batch.append(b)
                host.append(h)
                if B == 0:
                    _, d2, b2, _ = timed(lambda: eng.simulate_resident_removals(cand, mo, ms, persist=True, enc=after),
                                         "cae_simulate_resident_removals")
                    res_dev.append(d2)
                    res_batch.append(b2)
            h2d, d2h = int(st.h2d_bytes), int(st.d2h_bytes)
            match_ms = 0.0
            if B:
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    eng.plan_removals(plan, enc=after)
                    torch.cuda.synchronize()
                match_ms = sum(e.device_time_total for e in prof.key_averages() if "pdb_match_kernel" in e.key) / 1e3
            row = dict(nodes=N, pods_per_node=a.pods, candidates=len(cand), pdbs=B, card=name, power_limit=power,
                       removable=int((first["result"] == 0).sum()), call_ms=round(statistics.median(dev), 3),
                       batch_ms=round(statistics.median(batch), 3),
                       match_ms=round(match_ms, 3), host_ms=round(statistics.median(host), 3), h2d_bytes=h2d, d2h_bytes=d2h,
                       resident_call_ms=round(statistics.median(res_dev), 3) if res_dev else None,
                       resident_batch_ms=round(statistics.median(res_batch), 3) if res_batch else None, checked=checked)
            line = json.dumps(row)
            print(line, flush=True)
            if out:
                out.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
