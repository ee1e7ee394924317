"""Time cae_template_daemonsets: the DaemonSet pods of every node-group template in one call, against the host mirror.

For C3 / C5 template shapes at T templates and D DaemonSets (specs drawn from the snapshot's pod specs), three ways to get
the template pod lists a tick needs are timed with a host clock around calls that end in a stream synchronise:
  report   the call without apply (run_bits and run_count back on the host);
  apply    the call with apply: every template keeps the pods it had at the load and gets its DaemonSet pods after them
           (two DaemonSet sets alternate, so every call changes the lists);
  mirror   the host mirror: run_bits_encoded over every (template, DaemonSet), apply_run_bits, then cae_load_templates of
           the changed rows (the mirror is Python, not the shim's Go: a stand-in for the Go loop, not a measure of it).
--check compares the bits with the mirror and, after an apply, the engine's dense pass and Estimate() with a fresh load
of the objects the mirror states.  One JSON line per (config, T, D); the GPU name and power limit come first.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--templates", default="1000,5000,10000")
    ap.add_argument("--ds", default="10,50")
    ap.add_argument("--configs", default="3,5")
    ap.add_argument("--pods", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--mirror-reps", type=int, default=2)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import __graft_entry__ as g
    g.build()
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.daemonset import apply_run_bits, run_bits_encoded, unpack_rows
    from kubernetes_autoscaler_b200.encode import DaemonSetInputs
    from kubernetes_autoscaler_b200.engine import Engine

    def call(eng, ds, keep=None):
        """The C entry point alone (Engine.template_daemonsets also states the objects after an apply, in Python)."""
        di = DaemonSetInputs(ds_spec=ds, evaluate=None, running=None, keep=keep)
        bits = np.zeros((eng.enc.T, (len(ds) + 31) // 32), np.uint32)
        count = np.zeros(eng.enc.T, np.int32)
        t0 = time.perf_counter()
        rc = eng.lib.cae_template_daemonsets(eng.h, di.ptr(), bits.ctypes.data_as(C.c_void_p), count.ctypes.data_as(C.c_void_p))
        dt = time.perf_counter() - t0
        assert rc == 0, rc
        return dt, bits, count

    lines = [json.dumps({"card": card()})]
    print(lines[0], flush=True)
    eng, fresh = Engine(device=0), Engine(device=0) if args.check else None
    for config in [int(x) for x in args.configs.split(",")]:
        for T in [int(x) for x in args.templates.split(",")]:
            enc = synth.generate(config, pods=args.pods, templates=T)
            a, N = enc.arrays, enc.struct.num_cluster_nodes
            used = np.unique(np.concatenate([a["pend_spec"], a["node_pod_spec"]])).astype(np.int32)
            keep = np.diff(a["node_pod_off"][N:]).astype(np.int32)
            for D in [int(x) for x in args.ds.split(",")]:
                rng = np.random.default_rng(config * 100003 + T * 7 + D)
                sets = [used[rng.integers(0, len(used), D)] for _ in range(2)]
                row = {"config": config, "T": T, "D": D, "pods": args.pods}
                eng.load(enc)
                call(eng, sets[0])   # warm-up
                ts = []
                for _ in range(args.reps):
                    dt, bits, count = call(eng, sets[0])
                    ts.append(dt)
                row["report_ms"] = [round(1e3 * min(ts), 3), round(1e3 * float(np.median(ts)), 3), round(1e3 * max(ts), 3)]
                row["run_fraction"] = round(float(count.sum()) / max(T * D, 1), 4)
                if args.check:
                    want = run_bits_encoded(enc, sets[0])
                    assert np.array_equal(unpack_rows(bits, D), want), "run_bits differ from the mirror"
                    assert np.array_equal(count, want.sum(axis=1))
                ts = []
                for k in range(args.reps + 1):
                    dt = call(eng, sets[k % 2], keep)[0]
                    if k:   # the first apply warms the template-delta buffers
                        ts.append(dt)
                row["apply_ms"] = [round(1e3 * min(ts), 3), round(1e3 * float(np.median(ts)), 3), round(1e3 * max(ts), 3)]
                row["apply_h2d_bytes"], row["apply_d2h_bytes"] = int(eng.stats().h2d_bytes), int(eng.stats().d2h_bytes)
                if args.check:
                    last = sets[args.reps % 2]
                    after = apply_run_bits(enc, last, run_bits_encoded(enc, last), keep)[1]
                    fresh.load(after)
                    caps = np.full(T, 30, np.int32)
                    eng.enc = after
                    assert np.array_equal(eng.feasibility()[2], fresh.feasibility()[2]), "dense pass differs after apply"
                    for x, y in zip(eng.estimate_all(caps), fresh.estimate_all(caps)):
                        assert np.array_equal(x, y), "Estimate() differs after apply"
                ts = []
                for k in range(args.mirror_reps):
                    eng.load(enc)
                    t0 = time.perf_counter()
                    run = run_bits_encoded(enc, sets[k % 2])
                    delta, _ = apply_run_bits(enc, sets[k % 2], run, keep)
                    assert eng.load_templates(delta)
                    ts.append(time.perf_counter() - t0)
                row["mirror_ms"] = [round(1e3 * min(ts), 3), round(1e3 * float(np.median(ts)), 3), round(1e3 * max(ts), 3)]
                if args.check:
                    row["check"] = "ok"
                lines.append(json.dumps(row))
                print(lines[-1], flush=True)
    eng.close()
    if fresh is not None:
        fresh.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
