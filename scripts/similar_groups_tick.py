#!/usr/bin/env python
"""cae_similar_node_groups at T = 1 000 / 5 000 / 10 000 node groups, with C3 (E = 1 000) and C5 (E = 10 000) pod shapes and
families of 1 / 3 / 8 zones (synth.node_group_families).  Per shape, one JSON line:

  * device_ms: CUDA events on the engine's stream around the call (median of --reps after a warm-up; the group reasons
    are already valid, as after cae_estimate_all), first_ms: the first call after the load (group reasons computed in it);
  * host_ms: host wall time of the call (it ends in a stream synchronise), median;
  * d2h_bytes of the call against the T x E bytes of cae_feasibility_groups, the route that copies the exemplar matrix to
    the host for the subset test;
  * --check m: the first m base rows against the host mirror (tests/nodegroupset_harness.py); python_rows_ms is that
    mirror's CPU time per row, and python_all_rows_s its extrapolation to T rows.  Both are Python, not Go.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--templates", default="1000,5000,10000")
    ap.add_argument("--configs", default="3,5")
    ap.add_argument("--families", default="1,3,8")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--check", type=int, default=0, metavar="M")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.engine import Engine
    from kubernetes_autoscaler_b200.estimator import BasicIgnoredLabels, ScaleUpSimulation
    import nodegroupset_harness as h
    name, power = card()
    eng = Engine(device=0)
    stream = torch.cuda.ExternalStream(eng.stream())
    out = open(a.out, "w") if a.out else None
    for cfg in [int(x) for x in a.configs.split(",")]:
        for T in [int(x) for x in a.templates.split(",")]:
            for fam in [int(x) for x in a.families.split(",")]:
                infos, groups, ngs = synth.node_group_families(cfg, T, fam, seed=T + fam)
                sim = ScaleUpSimulation([], infos, groups, eng)
                res_sig, free_dims = sim.encoder.similarity_signatures(sim.templates)
                kw = dict(res_sig=res_sig, free_dims=free_dims, eligible=np.ones(T, np.uint8),
                          max_size=[ng.max_size for ng in ngs], target_size=[ng.target_size for ng in ngs],
                          ignored_keys=sim.encoder.label_key_ids(BasicIgnoredLabels))

                def timed():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    t0 = time.perf_counter()
                    r = eng.similar_node_groups(**kw)
                    t1 = time.perf_counter()
                    e1.record(stream)
                    e1.synchronize()
                    return r, e0.elapsed_time(e1), (t1 - t0) * 1e3
                (bits, count, limit), first_ms, _ = timed()
                dev, host = [], []
                for _ in range(a.reps):
                    r, d, hms = timed()
                    assert all(np.array_equal(x, y) for x, y in zip(r, (bits, count, limit)))
                    dev.append(d)
                    host.append(hms)
                row = dict(config="C%d" % cfg, templates=T, groups=len(groups), family=fam, card=name, power_limit=power,
                           device_ms=round(statistics.median(dev), 4), host_ms=round(statistics.median(host), 4),
                           first_ms=round(first_ms, 4), d2h_bytes=int(eng.stats().d2h_bytes),
                           feasibility_groups_d2h_bytes=T * len(groups), similar_pairs=int(count.sum()))
                if a.check:
                    sched = sim.schedulable_pod_groups()
                    cmp = h.CreateGenericNodeInfoComparator()
                    member = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :T]
                    t0 = time.perf_counter()
                    for t in range(min(a.check, T)):
                        ng = sim.ids[t]
                        want = h.ComputeSimilarNodeGroups(ng, h.FindSimilarNodeGroups(ng, infos, cmp), sched)
                        assert [sim.ids[s] for s in np.flatnonzero(member[t])] == want, (T, fam, t)
                    per_row = (time.perf_counter() - t0) / min(a.check, T)
                    row.update(checked_rows=min(a.check, T), python_rows_ms=round(per_row * 1e3, 2),
                               python_all_rows_s=round(per_row * T, 1))
                line = json.dumps(row)
                print(line, flush=True)
                if out:
                    out.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
