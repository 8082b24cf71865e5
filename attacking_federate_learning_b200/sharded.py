"""D-sharded multi-GPU aggregation: one process per GPU (torch.distributed), GPU r holds the column
block G[:, r*D/P:(r+1)*D/P].  Coordinate-wise rules (trimmed mean, mean, ALIE, Bulyan stage 2) need
no communication.  Krum / Bulyan need exactly one sum-all-reduce of the N x N float64 table of partial
squared distances (squared sums add across shards; the square root is taken after the reduce), after
which selection runs replicated and deterministically on every rank.

The per-shard arithmetic is delegated to a `kernels` object; the default binds the CUDA library.
(Tests inject a NumPy stand-in to exercise the sharding / collective logic on CPU with gloo.)
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist


def shard_bounds(dim: int, world: int, rank: int, align: int = 32):
    """Contiguous column block of `rank`, boundaries aligned to `align` columns (tile width)."""
    blocks = (dim + align - 1) // align
    b0 = blocks * rank // world
    b1 = blocks * (rank + 1) // world
    return min(b0 * align, dim), min(b1 * align, dim)


class NativeKernels:
    def __getattr__(self, name):
        from . import _device as dev
        return getattr(dev, name)

    def deviation_sums(self, G, corrupted_count, aggregated=None, krum_index=None):
        from . import batched
        return batched.attack_metrics(G, corrupted_count, aggregated=aggregated,
                                      krum_index=krum_index)["deviation_sums"]


class ShardedAggregator:
    def __init__(self, group=None, kernels=None):
        self.group = group
        self.k = kernels if kernels is not None else NativeKernels()
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self._buf = {}
        self._peer = None                 # PeerContext (NVLink peer-memory exchange) or None
        self._peer_error = None           # why the peer path is off (then NCCL all-reduce is used)

    # -- NVLink peer-memory exchange (csrc/xgpu.cu); falls back to the NCCL all-reduce if it cannot be set up
    def _peer_context(self, n, device):
        if self._peer_error is None and os.environ.get("AFL_XGPU", "1") == "0":
            self._peer_error = "disabled by AFL_XGPU=0"
        if self._peer_error is not None or not hasattr(self.k, "PeerContext"):
            return None
        if self._peer is not None and self._peer.n_max >= n:
            return self._peer
        ok = 1
        ctx = None
        try:
            if self._peer is not None:
                self._peer.close(); self._peer = None
            ctx = self.k.PeerContext(self.world, self.rank, max(n, 128), device)
            if self.world > 1:
                handles = [None] * self.world
                dist.all_gather_object(handles, ctx.handle(), group=self.group)
                ctx.connect(handles)
        except Exception as ex:          # pragma: no cover - depends on the box (IPC permissions, peer access)
            ok = 0
            self._peer_error = repr(ex)[:300]
        if self.world > 1:                # every rank must take the same path
            flag = torch.tensor([ok], device=device, dtype=torch.int32)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
            ok = int(flag.item())
        if not ok:
            self._peer_error = self._peer_error or "a peer rank could not map the exchange buffers"
            if ctx is not None:
                try:
                    ctx.close()
                except Exception:
                    pass
            return None
        self._peer = ctx
        return ctx

    # -- the single exchange step of the path
    def _allreduce_table(self, d2):
        if self.world > 1:
            dist.all_reduce(d2, op=dist.ReduceOp.SUM, group=self.group)
        return d2

    def distances(self, G_shard):
        return self.k.sqdist_to_dist(self._allreduce_table(self.k.sqdist_partial(G_shard)))

    def _buffers(self, n, device):
        key = (n, str(device))
        if self._buf.get("key") != key:
            self._buf = {"key": key, "d2": torch.empty((n, n), dtype=torch.float64, device=device),
                         "idx": torch.empty(1, dtype=torch.int32, device=device)}
        return self._buf["d2"], self._buf["idx"]

    def krum(self, G_shard, users_count, corrupted_count, return_index=False):
        if not return_index:
            assert users_count >= 2 * corrupted_count + 1, ('users_count>=2*corrupted_count + 3', users_count, corrupted_count)
        peer = self._peer_context(G_shard.shape[0], G_shard.device) if G_shard.is_cuda else None
        if peer is not None:
            # hot path (any world size, including 1): ONE FFI crossing: Gram -> publish -> Krum kernel on the ranks'
            # tables (peer-memory sum, sqrt, sort, score, argmin), index through mapped pinned memory, one stream
            # synchronisation
            idx = peer.krum(G_shard, users_count, corrupted_count)
        elif hasattr(self.k, "krum_from_sqdist"):
            # peer path off: two FFI crossings + the NCCL all-reduce, then the same Krum kernel on the summed d2 table;
            # persistent buffers, one 4-byte D2H sync
            d2, idx_dev = self._buffers(G_shard.shape[0], G_shard.device)
            self.k.sqdist_partial(G_shard, 0, d2)
            self._allreduce_table(d2)
            idx = int(self.k.krum_from_sqdist(d2, users_count, corrupted_count, idx_dev).item())
        else:                                            # kernels without krum_from_sqdist (the NumPy stand-in)
            idx = int(self.k.krum_select(self.distances(G_shard), users_count, corrupted_count).reshape(-1)[0].item())
        return idx if return_index else G_shard[idx]

    def bulyan(self, G_shard, users_count, corrupted_count, return_selection=False):
        assert users_count >= 4 * corrupted_count + 3
        peer = self._peer_context(G_shard.shape[0], G_shard.device) if (G_shard.is_cuda and self.world > 1) else None
        if peer is not None:
            d2, _ = self._buffers(G_shard.shape[0], G_shard.device)
            table = self.k.sqdist_to_dist(peer.allreduce_table(G_shard, d2))
        else:
            table = self.distances(G_shard)
        sel = self.k.bulyan_select(table, users_count, corrupted_count)
        out = self.k.trimmed_mean(G_shard, 2 * corrupted_count, row_index=sel)
        if len(sel) and int(sel[-1]) < 0:                # no eligible user in some round: defences.py:66 raises KeyError(-1)
            raise KeyError(-1)
        return (out, sel) if return_selection else out

    def trimmed_mean(self, G_shard, users_count, corrupted_count):
        return self.k.trimmed_mean(G_shard, corrupted_count)

    def no_defense(self, G_shard, users_count=None, corrupted_count=None):
        return self.k.mean(G_shard)

    def alie(self, G_shard, corrupted_count, num_std, write_rows=True, source_rows=None):
        """malicious.py:10-27 on this column shard: statistics over the malicious rows (rows 0..f-1, or
        `source_rows` = a [f, d_local] view of their honest gradients), crafted = mu - z*sigma, written back into
        rows 0..f-1 of the matrix when `write_rows` (what server.py:82-83 does with the aliased arrays)."""
        src = G_shard[:corrupted_count] if source_rows is None else source_rows
        bcast = G_shard if (write_rows and G_shard.dtype == torch.float32) else None
        crafted, _, _ = self.k.alie(src, num_std, bcast)
        return crafted

    def relative_deviation(self, G_shard, corrupted_count, aggregated=None, krum_index=None):
        """batched.attack_metrics' `rel_deviation` on column shards: G_shard is this rank's [B, N, d_local] block,
        `aggregated` its [B, d_local] slice of the aggregate (or `krum_index` the replicated int32 [B] indices).
        Each rank takes its shard's two float64 sums of squares per problem; they add across shards, so one
        all-reduce of the [B, 2] table and a square root give ||a - h|| / ||h|| over all D columns (fp32 [B]),
        identical on every rank."""
        sums = self._allreduce_table(self.k.deviation_sums(G_shard, corrupted_count, aggregated, krum_index))
        return torch.sqrt(sums[:, 0] / sums[:, 1]).float()

    def exchange_name(self):
        if self.world == 1:
            return "none"
        if self._peer is not None:
            return "NVLink peer-memory sum inside the Krum kernel (csrc/xgpu.cu, csrc/select.cu)"
        return "NCCL all-reduce" + (f" (peer path off: {self._peer_error})" if self._peer_error else "")

    def defend(self, name, G_shard, users_count, corrupted_count):
        return {"Krum": self.krum, "TrimmedMean": self.trimmed_mean, "NoDefense": self.no_defense,
                "Bulyan": self.bulyan}[name](G_shard, users_count, corrupted_count)

    def gather_output(self, out_shard, dim):
        """Optional: replicate the full [D] result on every rank (all_gather of the slices)."""
        if self.world == 1:
            return out_shard
        sizes = [shard_bounds(dim, self.world, r)[1] - shard_bounds(dim, self.world, r)[0] for r in range(self.world)]
        width = max(sizes)                                   # all_gather needs equal-sized pieces
        mine = torch.zeros(width, dtype=out_shard.dtype, device=out_shard.device)
        mine[:out_shard.numel()] = out_shard
        parts = [torch.empty(width, dtype=out_shard.dtype, device=out_shard.device) for _ in sizes]
        dist.all_gather(parts, mine, group=self.group)
        return torch.cat([p[:s] for p, s in zip(parts, sizes)])
