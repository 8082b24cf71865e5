"""world_size-2 gloo test (CPU) of ShardedAggregator.relative_deviation: each rank's per-problem float64 sums of
squares over its column block are all-reduced once and the square root is taken after the reduce.  The per-shard sums
are a NumPy stand-in, so this exercises the host logic of attacking_federate_learning_b200/sharded.py only."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ref_numpy as orc

FS = [2, 0, 5, 11]                     # per problem; 11 = no honest row


class NumpyKernels:
    """deviation_sums as batched.attack_metrics returns them: [B, 2] float64 (sum (a - h)^2, sum h^2) of this shard."""

    def deviation_sums(self, G, fs, aggregated=None, krum_index=None):
        out = np.empty((G.shape[0], 2))
        for b, Gb in enumerate(G.numpy()):
            if fs[b] >= len(Gb):
                out[b] = np.nan
                continue
            h = orc.no_defense(Gb[fs[b]:]).astype(np.float64)
            a = aggregated[b].numpy() if aggregated is not None else Gb[int(krum_index[b])]
            out[b] = ((a.astype(np.float64) - h) ** 2).sum(), (h ** 2).sum()
        return torch.from_numpy(out)


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _inputs(n, d):
    rng = np.random.default_rng(17)
    G = (0.1 * rng.standard_normal((len(FS), 1, d)) + rng.standard_normal((len(FS), n, d))).astype(np.float32)
    return G, G.mean(axis=1) + np.float32(0.01), np.array([3, 0, 10, 1], np.int32)


def _worker(rank, world, port, n, d, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from attacking_federate_learning_b200.sharded import ShardedAggregator, shard_bounds
    G, agg, idx = _inputs(n, d)
    c0, c1 = shard_bounds(d, world, rank)
    shard = torch.from_numpy(np.ascontiguousarray(G[:, :, c0:c1]))
    sa = ShardedAggregator(kernels=NumpyKernels())
    by_agg = sa.relative_deviation(shard, FS, aggregated=torch.from_numpy(np.ascontiguousarray(agg[:, c0:c1])))
    by_idx = sa.relative_deviation(shard, FS, krum_index=torch.from_numpy(idx))
    q.put((rank, by_agg.numpy(), by_idx.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_relative_deviation_matches_unsharded():
    world, n, d = 2, 11, 333
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, d, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {r: (a, i) for r, a, i in (q.get(timeout=120) for _ in range(world))}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0

    G, agg, idx = _inputs(n, d)
    for b, f in enumerate(FS):
        for k, a in enumerate((agg[b], G[b, idx[b]])):
            if f >= n:
                assert all(np.isnan(got[r][k][b]) for r in range(world))
                continue
            h = orc.no_defense(G[b, f:]).astype(np.float64)
            want = np.linalg.norm(a.astype(np.float64) - h) / np.linalg.norm(h)
            for r in range(world):
                assert got[r][k].dtype == np.float32
                assert abs(got[r][k][b] - want) <= 1e-6 * want, (b, k, r)
            assert got[0][k][b] == got[1][k][b]                                # replicated, identical on every rank
