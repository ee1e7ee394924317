"""N>1 path on CPU: world_size-2 gloo.  The ranks shard pods (dense pass) / templates (pack) exactly
like the engine does and assemble the result with ONE sum all-reduce each; the per-shard numbers come
from the CPU oracle here (the GPU parity of every rank's shard is covered by tests/test_gpu_shards.py)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from kubernetes_autoscaler_b200 import synth
from kubernetes_autoscaler_b200.engine import shard_pods, shard_templates


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import pyoracle
    enc = synth.generate(2, pods=3000, templates=64)
    # dense pass: pods sharded, int32[T] fit histogram all-reduced
    pb, pe = shard_pods(enc.P, rank, world)
    reasons, _ = pyoracle.feasibility_dense(enc, p_range=(pb, pe))
    hist = torch.from_numpy((reasons == 0).sum(axis=1).astype(np.int32))
    dist.all_reduce(hist)
    # pack: templates sharded, zero-filled int32[2T] all-reduced
    tb, te = shard_templates(enc.T, rank, world)
    caps = np.full(enc.T, 50, np.int32)
    nc, pc, sched, _, _ = pyoracle.estimate_all(enc, caps, t_range=(tb, te))
    # expander: least-waste scores of the own templates, 0.0 elsewhere; a float64 sum all-reduce assembles them exactly
    full_nc, full_pc, full_sched = np.zeros(enc.T, np.int32), np.zeros(enc.T, np.int32), np.zeros((enc.T, enc.E), np.int32)
    full_nc[tb:te], full_pc[tb:te], full_sched[tb:te] = nc, pc, sched
    _, own_waste = pyoracle.expander(enc, [0], full_nc, full_pc, full_sched)
    waste = torch.zeros(enc.T, dtype=torch.float64)
    waste[tb:te] = torch.from_numpy(own_waste[tb:te])
    dist.all_reduce(waste)
    counts = torch.zeros(2 * enc.T, dtype=torch.int32)
    counts[tb:te] = torch.from_numpy(nc)
    counts[enc.T + tb:enc.T + te] = torch.from_numpy(pc)
    dist.all_reduce(counts)
    bits = np.packbits(reasons == 0, axis=1, bitorder="little")
    np.save(os.path.join(out_dir, "bits%d.npy" % rank), bits)
    if rank == 0:
        np.save(os.path.join(out_dir, "hist.npy"), hist.numpy())
        np.save(os.path.join(out_dir, "counts.npy"), counts.numpy())
        np.save(os.path.join(out_dir, "waste.npy"), waste.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_shard_boundaries():
    for P in (0, 1, 31, 32, 33, 1000, 100_000, 1_000_003):
        for W in (1, 2, 3, 4, 8):
            cuts = [shard_pods(P, r, W) for r in range(W)]
            assert cuts[0][0] == 0 and cuts[-1][1] == P
            for (b0, e0), (b1, e1) in zip(cuts, cuts[1:]):
                assert e0 == b1 and b1 % 32 == 0
            tc = [shard_templates(P, r, W) for r in range(W)]
            assert tc[0][0] == 0 and tc[-1][1] == P and all(a[1] == b[0] for a, b in zip(tc, tc[1:]))


def test_two_rank_gloo_assembles_the_single_rank_result(tmp_path, oracle):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    enc = synth.generate(2, pods=3000, templates=64)
    want, _ = oracle.feasibility_dense(enc)
    assert np.array_equal(np.load(tmp_path / "hist.npy"), (want == 0).sum(axis=1))
    caps = np.full(enc.T, 50, np.int32)
    nc, pc, sched, _, _ = oracle.estimate_all(enc, caps)
    assert np.array_equal(np.load(tmp_path / "counts.npy"), np.concatenate([nc, pc]))
    # the sharded expander: all-reduced waste vector is bit-identical, and the host chain (cae_expander_chain, no GPU
    # needed) picks the same options as the single-rank expander
    from kubernetes_autoscaler_b200.engine import expander_chain
    waste = np.load(tmp_path / "waste.npy")
    for chain in ([0], [0, 1, 2], [2, 0], [1]):
        omask, owaste = oracle.expander(enc, chain, nc, pc, sched)
        assert np.array_equal(waste, owaste)
        assert np.array_equal(expander_chain(chain, nc, pc, waste), omask), chain
    # word-aligned shards: bit rows concatenate into the full matrix
    full = np.concatenate([np.load(tmp_path / ("bits%d.npy" % r)) for r in range(world)], axis=1)
    assert np.array_equal(np.unpackbits(full, axis=1, bitorder="little")[:, :enc.P].astype(bool), want == 0)
