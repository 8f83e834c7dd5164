"""Multi-GPU retrieval: the database is sharded row-wise, one process per GPU (SURVEY.md 8e).

Rank g owns the contiguous rows [g*N/G, (g+1)*N/G) - the descriptors it extracted - and searches them with
dirb200_index_search (global indices = local row + offset).  The only data-path exchange is ONE all-gather of
the per-shard top-k lists ((fp64 score, int64 index)[Q][k] per rank, 16*Q*k bytes) followed by the same k-way
merge on every rank; alpha query expansion adds ONE all-reduce of the Q x D partial neighbour sums.  The
reference's analogue is nn.DataParallel (dirtorch/utils/common.py:155); extraction needs no communication.

torch.distributed is plumbing only (NCCL over NVLink on GPUs, gloo on CPU for the unit tests).
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_rows(n_rows: int, world: int, rank: int):
    """Contiguous row range of `rank`: [start, end)."""
    return (n_rows * rank) // world, (n_rows * (rank + 1)) // world


def shard_quota(k: int, shard_sizes) -> int:
    """Per-shard selection depth c of the two-phase search: shard g reports its min(c, N_g)-th best score, and the
    MINIMUM of the reports is a lower bound on the global k-th best only if the shards can certify k rows between
    them, i.e.  sum_g min(c, N_g) >= min(k, sum_g N_g).  This returns the smallest such c: ceil(k / G) when every
    shard holds at least that many rows, more when some shards are small or empty (c = k always satisfies it)."""
    sizes = [int(n) for n in shard_sizes]
    need = min(int(k), sum(sizes))
    c = max(1, -(-int(k) // max(1, len(sizes))))
    while c < k and sum(min(c, n) for n in sizes) < need:
        c += 1
    return min(c, int(k))


def sort_thresholds(s: torch.Tensor, t_q: torch.Tensor) -> torch.Tensor:
    """Values s grouped by query (t_q non-decreasing) -> the same groups, each sorted in descending order."""
    order = torch.sort(s, descending=True, stable=True).indices
    return s[order][torch.sort(t_q[order], stable=True).indices]


def all_gather_packed(packed: torch.Tensor, group=None) -> torch.Tensor:
    """packed (2,Q,k) int64 per rank -> (G,2,Q,k); a single collective."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return packed.unsqueeze(0)
    flat = torch.empty(world * packed.numel(), dtype=packed.dtype, device=packed.device)
    dist.all_gather_into_tensor(flat, packed.contiguous().view(-1), group=group)
    return flat.view((world,) + tuple(packed.shape))


class ShardedIndex:
    """Row shard of the database on this rank + the cross-rank top-k exchange."""

    def __init__(self, db32_local: torch.Tensor, row_offset: int, group=None, db16_local=None):
        from . import ops
        self.ops = ops
        self.group = group
        self.row_offset = int(row_offset)
        self.local = ops.Index(db32_local, index_offset=row_offset, db16=db16_local)
        self.local.set_option("retries", 2)      # a rank cannot re-run alone (collectives): one more gated retry pass up front
        self.xchg = None                         # peer-memory exchange window (enable_peer_exchange)
        self._qmax = {}                          # k -> query block of the collective path (_max_queries)
        # row counts of all shards (one small all-gather at construction, not on the search path): the selection depth
        # of the two-phase search depends on them, see shard_quota
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world > 1:
            mine = torch.tensor([self.local.n], dtype=torch.int64, device=db32_local.device)
            sizes = torch.empty(world, dtype=torch.int64, device=db32_local.device)
            dist.all_gather_into_tensor(sizes, mine, group=group)
            self.shard_sizes = [int(v) for v in sizes.tolist()]
        else:
            self.shard_sizes = [int(self.local.n)]
        self.local.n_global = sum(self.shard_sizes)   # allow sets number the rows of the whole database

    def enable_peer_exchange(self, max_q: int = 1024, max_k: int = 128):
        """Switch search() to the peer-memory protocol (dirb200_index_search_sharded): the MIN of the selection thresholds
        and the gather of the per-shard lists are done by the search kernels themselves with stores into the other ranks'
        exchange windows over NVLink - no NCCL call on the search path.  One process per GPU of ONE box (CUDA IPC); the
        only collective is the one-off all-gather of the 64-byte IPC handles here.  Collective call.  Searches with more
        than max_q queries or k > max_k keep using the torch.distributed collectives (same results); call
        disable_peer_exchange() (collective) before the ranks drop their indices."""
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        rank = dist.get_rank(self.group) if dist.is_initialized() else 0
        dev = self.local.db32.device
        x = self.ops.Exchange(dev.index or 0, world, rank, max_q, max_k)
        if world > 1:
            mine = torch.frombuffer(bytearray(x.ipc_handle()), dtype=torch.uint8).to(dev)
            allh = torch.empty(world * 64, dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(allh, mine, group=self.group)
            blob = bytes(allh.cpu().numpy().tobytes())
            x.open([blob[64 * g: 64 * (g + 1)] for g in range(world)])
            dist.barrier(group=self.group)          # every window is mapped everywhere before the first search writes to it
        else:
            self.ops.Exchange.open_local([x])
        self.xchg = x
        return self

    def disable_peer_exchange(self):
        """Tear the exchange down in the order CUDA IPC requires: every rank unmaps the peers' windows, barrier, every rank
        frees its own window.  Collective call; search() goes back to the torch.distributed collectives."""
        x, self.xchg = self.xchg, None
        if x is None:
            return self
        x.close_peers()
        if dist.is_initialized() and dist.get_world_size(self.group) > 1:
            dist.barrier(group=self.group)
        x.close()
        return self

    @classmethod
    def from_store(cls, store, device, group=None, chunk_rows: int = 65536):
        """Load this rank's row range of an on-disk descriptor store (store.py) and index it.  The split is
        ``shard_rows`` over the CURRENT world size, whatever shard files the store was written in."""
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        rank = dist.get_rank(group) if dist.is_initialized() else 0
        start, end = shard_rows(len(store), world, rank)
        d32, d16 = store.load_rows_to_device(start, end, device, chunk_rows)
        return cls(d32, start, group, db16_local=d16)

    def search_local(self, q32: torch.Tensor, k: int):
        packed = torch.empty((2, q32.shape[0], k), dtype=torch.int64, device=q32.device)
        self.local.search(q32, k, out=packed)
        return packed

    def search(self, q32: torch.Tensor, k: int, check: bool = True, allow=None):
        """Global exact top-k.  Phase 1 on every shard (tensor-core passes) -> MIN all-reduce of the per-query
        selection thresholds (4*Q bytes: the local c-th best scores, c = shard_quota(k, shard sizes) = ceil(k/G) for
        evenly filled shards, bound the global k-th best, so each shard re-scores only ~k/G rows) -> phase 2 (exact
        re-scoring) -> one all-gather of the per-shard lists -> merge.  Returns (scores fp64, idx int64), (Q,k).

        Nothing on this path waits for the GPU except the status check of the local shard (candidate overflow that the
        device-side retry passes could not resolve).  check=True collects it before returning; check=False leaves it
        to the next search() / an explicit check() so that the host can enqueue the next search while this one runs.

        allow: filtered search (DESIGN.md section 4.13, rule F6) - the same allow set on every rank, in global row
        numbering: (W,) int32 words shared by every query or (Q, W) one per query, W = ceil(total rows / 32)."""
        world = dist.get_world_size(self.group) if dist.is_initialized() else 1
        filt = {} if allow is None else {"allow": allow}
        if world == 1:
            self.local.set_option("deferred_check", 0 if check else 1)
            return self.local.search(q32, k, **filt)         # the shard's ordered list IS the result: no merge pass
        if allow is not None:
            self.local._allow_ld(allow, q32.shape[0])        # bad arguments raise before any device call
        self.local.set_option("deferred_check", 1)
        k_shard = shard_quota(k, self.shard_sizes)
        x = self.xchg
        if x is not None and q32.shape[0] <= x.max_q and k <= x.max_k:
            out = self.local.search_sharded(x, q32, k, k_shard, **filt)   # thresholds + lists travel through peer memory
            if check:
                self.local.check()
            return out
        qb = self._max_queries(k)
        parts = []
        for q0 in range(0, q32.shape[0], qb):               # query blocks whose workspace fits every shard's budget
            qc = q32[q0:q0 + qb].contiguous()
            if allow is not None:
                filt["allow"] = allow if allow.dim() == 1 else allow[q0:q0 + qb]
            sel = self.local.search_begin(qc, k, k_shard, **filt)
            dist.all_reduce(sel, op=dist.ReduceOp.MIN, group=self.group)
            packed = torch.empty((2, qc.shape[0], k), dtype=torch.int64, device=q32.device)
            self.local.search_finish(qc, k, sel, out=packed)
            gathered = all_gather_packed(packed, self.group)
            parts.append(self.ops.topk_merge_packed(gathered, k))
        out = parts[0] if len(parts) == 1 else (torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]))
        if check:
            self.local.check()
        return out

    def _max_queries(self, k: int) -> int:
        """Query block of a depth-k search: the smallest search_max_queries(k) over the shards (one MIN all-reduce the
        first time each k is seen; every rank calls search() with the same k, so the ranks fill the cache in step)."""
        if k not in self._qmax:
            t = torch.tensor([self.local.search_max_queries(k)], dtype=torch.int64, device=self.local.db32.device)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
            self._qmax[k] = int(t.item())
        return self._qmax[k]

    def check(self):
        """Status of the last search(check=False)."""
        self.local.check()

    def rank_counts(self, q32: torch.Tensor, t_off, t_rows, t_flags):
        """Exact scores of the labelled rows and the number of database rows ranking before each flagged one, over the
        WHOLE sharded database: each shard scores the targets it owns (one SUM all-reduce of T doubles), counts its own
        rows that rank before each target (one SUM all-reduce of T int64) - SURVEY 8e.  Returns CUDA tensors."""
        import numpy as np
        off = np.ascontiguousarray(t_off, dtype=np.int32)
        dev = q32.device
        t_q = torch.from_numpy(np.repeat(np.arange(q32.shape[0], dtype=np.int32), np.diff(off))).to(dev)
        rows = torch.as_tensor(np.ascontiguousarray(t_rows, dtype=np.int64)).to(dev)
        flags = torch.as_tensor(np.ascontiguousarray(t_flags, dtype=np.uint8)).to(dev)
        multi = dist.is_initialized() and dist.get_world_size(self.group) > 1
        sc = self.local.target_scores(q32, t_q, rows)
        if multi:
            dist.all_reduce(sc, op=dist.ReduceOp.SUM, group=self.group)      # exactly one shard contributes a non-zero
        above = self.local.rank_count(q32, off, rows, flags, sc)
        if multi:
            dist.all_reduce(above, op=dist.ReduceOp.SUM, group=self.group)
        return sc, above

    def count_ge(self, q32: torch.Tensor, t_off, t_rows, skip_row=None):
        """Label AP counts over the WHOLE sharded database.  t_off int32 (Q+1,) / t_rows int64 (T,) CUDA tensors: the
        positives of each query (global indices).  Each shard scores the positives it owns (one SUM all-reduce of T
        doubles); the fp32 roundings, sorted descending within each query, are the thresholds; each shard counts its
        own rows reaching them (one SUM all-reduce of T int64).  Returns (thresholds fp32 (T,), counts int64 (T,)) in
        the sorted order, CUDA tensors."""
        t_q = torch.repeat_interleave(torch.arange(q32.shape[0], dtype=torch.int32, device=q32.device),
                                      (t_off[1:] - t_off[:-1]).long())
        multi = dist.is_initialized() and dist.get_world_size(self.group) > 1
        sc = self.local.target_scores(q32, t_q, t_rows)
        if multi:
            dist.all_reduce(sc, op=dist.ReduceOp.SUM, group=self.group)      # exactly one shard contributes a non-zero
        thr = sort_thresholds(sc.float(), t_q)
        count = self.local.count_ge(q32, t_off, thr, skip_row)
        if multi:
            dist.all_reduce(count, op=dist.ReduceOp.SUM, group=self.group)
        return thr, count

    def expand_queries(self, q32: torch.Tensor, k: int, alpha: float, check: bool = True):
        """alpha-QE (test_dir.py:24-44) over the sharded database: global top-k, each rank sums the neighbours it
        owns, one all-reduce, add the query, normalise."""
        scores, idx = self.search(q32, k, check=check)
        partial = self.ops.aqe_expand(q32, self.local.db32, idx, scores, alpha, partial=True,
                                      row_offset=self.row_offset, n_rows=self.local.n)
        if dist.is_initialized() and dist.get_world_size(self.group) > 1:
            dist.all_reduce(partial, op=dist.ReduceOp.SUM, group=self.group)
        # normalize(q + sum) == normalize(mean([q, sum])): reuse the scale-pooling kernel
        return self.ops.pool_scales([partial, q32], "mean", l2=True)
