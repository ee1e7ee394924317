#!/usr/bin/env python
"""Small end-to-end workload for compute-sanitizer (SURVEY §5: memcheck / racecheck evidence for the kernels that use
self-cleaning accumulators, last-block election, shared-memory state and block-wide barriers):

    compute-sanitizer --tool memcheck  python scripts/sanitize.py
    compute-sanitizer --tool racecheck python scripts/sanitize.py

Dense pass (K1, both variants), Estimate() of every template (K0 + K3: plain closed form, capacity form with the cluster
fallback, per-pod loop), expander scores, the filter-out-schedulable pass, a scale-down batch (cae_simulate_removals), a cluster-node delta
(cae_load_nodes), a cluster-node churn (cae_load_node_churn), new pod specs (cae_load_pods) and the similar node groups (cae_similar_node_groups) — on miniatures of C2, C3 and C4 — each checked
against the CPU oracle so that a "clean" run also means "correct results under the tool"."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np  # noqa: E402


def main():
    import __graft_entry__ as ge
    ge.build()
    from kubernetes_autoscaler_b200 import synth
    from kubernetes_autoscaler_b200.engine import Engine, unpack_bits
    from kubernetes_autoscaler_b200.estimator import ScaleUpSimulation
    import nodegroupset_harness as h
    from oracle import pyoracle
    eng = Engine(device=0, want_reasons=True)
    for cfg, kw in ((2, dict(pods=3000, templates=40)), (3, dict(pods=2500, templates=24, cluster_nodes=48)),
                    (4, dict(pods=3000, templates=20, cluster_nodes=40))):
        enc = synth.generate(cfg, **kw)
        eng.load(enc)
        bits, reasons, count = eng.feasibility()
        want, _ = pyoracle.feasibility_dense(enc)
        assert np.array_equal(reasons, want) and np.array_equal(unpack_bits(bits, enc.P), want == 0)
        for cap in (30, 0):
            caps = np.full(enc.T, cap, np.int32)
            nc, pc, sched, order = eng.estimate_all(caps)
            onc, opc, osched, oorder, _ = pyoracle.estimate_all(enc, caps)
            assert np.array_equal(nc, onc) and np.array_equal(pc, opc) and np.array_equal(sched, osched) and np.array_equal(order, oorder)
        mask, waste = eng.expander_best([0, 1, 2], nc, pc)
        assert eng.load_pending(enc)
        eng.feasibility()
        if enc.struct.num_cluster_nodes:
            order_p = np.arange(min(enc.P, 600), dtype=np.int32)
            got = eng.filter_schedulable(order_p)
            ref = pyoracle.filter_schedulable(enc, order_p)
            assert np.array_equal(got[0], ref[0]) and got[1:] == ref[1:]
            # cluster-node delta (cae_load_nodes: row scatter, CSR rebuild, dirty-column class matrix, counter recount)
            delta, pending = synth.node_churn(enc, cfg, 12)
            assert eng.load_nodes(delta) and eng.load_pending(pending)
            after = pending.apply_node_delta(delta)
            eng.enc = after
            _, reasons, _ = eng.feasibility()
            assert np.array_equal(reasons, pyoracle.feasibility_dense(after)[0])
            caps = np.full(after.T, 30, np.int32)
            got_e, ref_e = eng.estimate_all(caps), pyoracle.estimate_all(after, caps)
            assert all(np.array_equal(x, y) for x, y in zip(got_e, ref_e[:4]))
            got = eng.filter_schedulable(order_p)
            ref = pyoracle.filter_schedulable(after, order_p)
            assert np.array_equal(got[0], ref[0]) and got[1:] == ref[1:]
            # scale-down batch (cae_simulate_removals): every cluster node a candidate, each listing its own slice of pending
            # pods, persisted; the filter pass on the same load is unchanged afterwards
            n = enc.struct.num_cluster_nodes
            cand = np.arange(n, dtype=np.int32)
            move_off = np.minimum(np.arange(n + 1, dtype=np.int32) * 4, len(order_p)).astype(np.int32)
            eng.simulate_removals(cand, move_off, order_p[:move_off[-1]], persist=True)
            got = eng.filter_schedulable(order_p)
            assert np.array_equal(got[0], ref[0]) and got[1:] == ref[1:]
            # cluster-node churn (cae_load_node_churn: column gather, CSR rebuild, domains, full class matrix, recount)
            churn, pending = synth.node_scale(after, cfg, 4, 4, 6)
            assert eng.load_node_churn(churn) and eng.load_pending(pending)
            after = pending.apply_node_churn(churn)
            eng.enc = after
            _, reasons, _ = eng.feasibility()
            assert np.array_equal(reasons, pyoracle.feasibility_dense(after)[0])
            caps = np.full(after.T, 30, np.int32)
            got_e, ref_e = eng.estimate_all(caps), pyoracle.estimate_all(after, caps)
            assert all(np.array_equal(x, y) for x, y in zip(got_e, ref_e[:4]))
            got = eng.filter_schedulable(order_p)
            ref = pyoracle.filter_schedulable(after, order_p)
            assert np.array_equal(got[0], ref[0]) and got[1:] == ref[1:]
            # new pod specs and a new pending list (cae_load_pods: spec tails appended, the pending-side derivation rerun)
            pdelta = synth.pod_churn(after, cfg, 3, 3)
            after = after.apply_pod_delta(pdelta)
            assert eng.load_pods(pdelta, after) == 0
            _, reasons, _ = eng.feasibility()
            assert np.array_equal(reasons, pyoracle.feasibility_dense(after)[0])
            caps = np.full(after.T, 30, np.int32)
            got_e, ref_e = eng.estimate_all(caps), pyoracle.estimate_all(after, caps)
            assert all(np.array_equal(x, y) for x, y in zip(got_e, ref_e[:4]))
            order_p = np.arange(min(after.P, 600), dtype=np.int32)
            got = eng.filter_schedulable(order_p)
            ref = pyoracle.filter_schedulable(after, order_p)
            assert np.array_equal(got[0], ref[0]) and got[1:] == ref[1:]
        # similar node groups (cae_similar_node_groups: operand / bit-row prep, the pair kernel's staged tiles and ballots)
        infos, groups, ngs = synth.node_group_families(cfg, 45, 4, seed=cfg, groups=40)
        sim = ScaleUpSimulation([], infos, groups, eng)
        got = sim.similar_node_groups(ngs)
        sched, cmp = sim.schedulable_pod_groups(), h.CreateGenericNodeInfoComparator()
        assert got == {t: h.ComputeSimilarNodeGroups(t, h.FindSimilarNodeGroups(t, infos, cmp), sched) for t in sim.ids}
        print("config", cfg, "ok: nodes", int(nc.sum()), "pods", int(pc.sum()), flush=True)
    eng.close()
    print("sanitize workload ok")


if __name__ == "__main__":
    main()
