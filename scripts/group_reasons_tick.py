#!/usr/bin/env python
"""cae_group_reasons at the C3 (5 000 templates, 1 000 groups) and C5 (10 000 templates, 10 000 groups) shapes, against the
route it replaces: cae_feasibility_groups plus the copy of the [T][E] reason matrix to the host.  Per config, one JSON line:

  * counts_ms / counts_first_ms: CUDA events on the engine's stream around group_reasons() (median of --reps after a
    warm-up; the group reasons are valid, as after cae_estimate_all) and the first call after the load (group reasons
    computed in it); detail_ms: the same with the [T][E] detail copied back;
  * matrix_ms: cae_feasibility_groups (recomputes the reasons and copies T x E bytes), median;
  * host_ms: host wall time of the counts call (it ends in a stream synchronise), median;
  * d2h_bytes of each route (cae_stats for the counts and detail calls, T x E for the matrix route).
The outputs of the counts call are checked against a numpy reduction of the matrix route's reasons where no Fit or
PreFilter split is needed (the totals per group).  The card name and power limit are read in the same run."""
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
    ap.add_argument("--configs", default="3,5")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import capi, synth
    from kubernetes_autoscaler_b200.engine import Engine
    name, power = card()
    eng = Engine(device=0)
    stream = torch.cuda.ExternalStream(eng.stream())
    out = open(a.out, "w") if a.out else None
    fit = capi.CONST["CAE_R_FIT"]

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        r = fn()
        t1 = time.perf_counter()
        e1.record(stream)
        e1.synchronize()
        return r, e0.elapsed_time(e1), (t1 - t0) * 1e3

    for cfg in [int(x) for x in a.configs.split(",")]:
        enc = synth.generate(cfg)
        T, E = enc.T, enc.E
        eng.load(enc)
        (sched, counts, _), first_ms, _ = timed(lambda: eng.group_reasons())
        dev, host, det, mat = [], [], [], []
        for _ in range(a.reps):
            r, d, h = timed(lambda: eng.group_reasons())
            assert np.array_equal(r[0], sched) and np.array_equal(r[1], counts)
            dev.append(d)
            host.append(h)
        d2h_counts = int(eng.stats().d2h_bytes)
        for _ in range(max(a.reps // 4, 3)):
            r, d, _ = timed(lambda: eng.group_reasons(want_detail=True))
            det.append(d)
        d2h_detail = int(eng.stats().d2h_bytes)
        for _ in range(max(a.reps // 4, 3)):
            reasons, d, _ = timed(eng.feasibility_groups)
            mat.append(d)
        # the totals the matrix route gives: non-Fit codes and the Fit key per group, and eg.Schedulable
        assert np.array_equal(sched, ((reasons == 0).any(axis=0) & (np.diff(enc.arrays["group_off"]) > 0)).astype(np.uint8))
        assert np.array_equal(counts[:, fit], (reasons == fit).sum(axis=0))
        row = dict(config="C%d" % cfg, templates=T, groups=E, card=name, power_limit=power,
                   counts_ms=round(statistics.median(dev), 4), counts_first_ms=round(first_ms, 4),
                   host_ms=round(statistics.median(host), 4), detail_ms=round(statistics.median(det), 4),
                   matrix_ms=round(statistics.median(mat), 4), d2h_bytes_counts=d2h_counts, d2h_bytes_detail=d2h_detail,
                   d2h_bytes_matrix=T * E)
        line = json.dumps(row)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
    eng.close()


if __name__ == "__main__":
    main()
