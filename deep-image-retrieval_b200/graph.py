"""Graph search over a pruned kNN graph of the database (extension; DESIGN.md section 4.12, rules G1-G8).

The graph keeps, for every row, `degree` edges chosen from its exact kNN list: the neighbours reachable without a
detour through a closer neighbour first, then reverse edges, as in CAGRA.  A query starts from its best rows among a
fixed sample and expands the best unexpanded rows of its running top-`itopk` list until none is left or `max_iter`
iterations have run (one CTA per query, csrc/graph.cu).  The result has an exact definition: the exact top-k of the set
V(q) of rows the traversal visited, with the scores and order of ``ops.Index.search``; V(q) is a deterministic function
of the data, the graph and the parameters.  ``tests/graph_model.py`` restates the rules in numpy.
"""
from __future__ import annotations

import numpy as np
import torch

from . import inputs, lib, ops
from .ivf import InvertedLists

MAX_K = 128             # the prune kernel's longest kNN list (build_k)
MAX_DEGREE = 128
SEARCH_DEFAULTS = dict(itopk=128, width=1, max_iter=256, n_seeds=16)


def smem_bytes(n_seeds, itopk, width, degree, max_iter):
    """Shared memory of one query of the search kernel (its visited table, B twice, the batch of new rows)."""
    return int(lib.raw("dirb200_graph_search_smem_bytes")(n_seeds, itopk, width, degree, max_iter))


def max_iter_limit(limit, n_seeds, itopk, width, degree):
    """The largest max_iter whose search fits `limit` bytes of shared memory per block (-1: none does)."""
    if smem_bytes(n_seeds, itopk, width, degree, 0) > limit:
        return -1
    lo, hi = 0, 1
    while smem_bytes(n_seeds, itopk, width, degree, hi) <= limit:
        lo, hi = hi, 2 * hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if smem_bytes(n_seeds, itopk, width, degree, mid) <= limit else (lo, mid)
    return lo


def _remove_self(idx, K):
    """Rule G2: each row's list of K + 1 entries without the row itself, or without its last entry when the row is not
    in it -> int32 (N, K)."""
    n = idx.shape[0]
    idx = idx[:, :K + 1]
    me = idx == torch.arange(n, device=idx.device)[:, None]
    last = torch.zeros_like(me)
    last[:, K] = True
    drop = torch.where(me.any(1, keepdim=True), me, last)
    return idx[~drop].view(n, K).to(torch.int32).contiguous()


class GraphIndex:
    """GraphIndex(X, degree=32, build_k=64, n_entry=4096, seed=0, knn=None, graph=None): X (N, D) unit rows (a CUDA
    tensor, a host array / memmap or a DescriptorStore), zero-padded to a multiple of 64 columns.

    The build takes every row's exact top-build_k list (rule G2: from ops.Index(X).search(X, build_k + 1), or from
    knn=(scores, idx) in that format, -1 entries allowed), keeps the `degree` entries with the fewest detours (G3, G4)
    and merges in reverse edges (G5).  degree <= 128, build_k <= 128.  graph= takes a saved graph_ instead (int (N,
    degree), entries in [-1, N)), so a build can be reused.  The entry sample (G6) is min(N, n_entry) rows drawn by
    numpy.random.default_rng(seed) without replacement, sorted.

    After the build: graph_ int32 (N, degree), entry_ int64 (CUDA tensors) and n_components_, the number of weakly
    connected components of the graph (a query can only reach rows of the components its seeds lie in)."""

    def __init__(self, X, degree=32, build_k=64, n_entry=4096, seed=0, knn=None, graph=None, device=None):
        self.dim = inputs.Rows(X).d
        with torch.cuda.device(inputs.device(device, X)):      # every launch of the build runs on that device
            self._setup(inputs.rows64(X), degree, build_k, n_entry, seed, knn, graph)

    def _setup(self, x, degree, build_k, n_entry, seed, knn, graph):
        n = x.shape[0]
        if n < 1:
            raise ValueError("need at least one row")
        if n >= 1 << 31:
            raise ValueError("at most 2^31 - 1 rows (got %d)" % n)
        inputs.check_unit(x, "X")
        self.x = x
        self.degree = inputs.check_int(degree, "degree", 1, MAX_DEGREE)
        self.build_k = min(inputs.check_int(build_k, "build_k", 1, MAX_K), n - 1)
        n_entry = inputs.check_int(n_entry, "n_entry")
        dev = x.device
        rng = np.random.default_rng(seed)
        self.entry_ = torch.from_numpy(np.sort(rng.choice(n, min(n, n_entry), replace=False))).to(dev)
        self._entry = ops.Index(x[self.entry_].contiguous())
        self.build_ms_ = {}
        if graph is not None:
            self.graph_ = self._check_graph(graph)
        else:
            self.graph_ = self._build(knn)
        g = self.graph_.view(-1).long()
        ok = g >= 0
        off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(ok.view(n, -1).sum(1), 0, out=off[1:])
        labels = ops.join_components(off, g[ok].contiguous(), n)
        self.n_components_ = int((labels == torch.arange(n, device=dev)).sum())
        self._stats = {}

    def _check_graph(self, graph):
        g = torch.as_tensor(graph).to(self.x.device)
        n = self.x.shape[0]
        if g.dim() != 2 or tuple(g.shape) != (n, self.degree):
            raise ValueError("graph must have shape (%d, %d) (got %s)" % (n, self.degree, tuple(g.shape)))
        if g.dtype.is_floating_point or g.dtype == torch.bool:
            raise ValueError("graph must hold integer rows (got %s)" % g.dtype)
        if g.numel() and (int(g.min()) < -1 or int(g.max()) >= n):
            raise ValueError("graph entries must lie in [-1, %d)" % n)
        return g.to(torch.int32).contiguous()

    def _knn(self, knn):
        """Rule G2 -> int32 (N, build_k)."""
        n, K = self.x.shape[0], self.build_k
        if knn is None:
            exact = ops.Index(self.x)
            try:
                idx = exact.search(self.x, K + 1)[1]
            finally:
                exact.close()
            return _remove_self(idx, K)
        idx = torch.as_tensor(knn[1]).to(self.x.device)
        if idx.dim() != 2 or idx.shape[0] != n or idx.shape[1] < K + 1:
            raise ValueError("knn rows must be (%d, >= %d) (got %s)" % (n, K + 1, tuple(idx.shape)))
        if idx.dtype.is_floating_point or idx.dtype == torch.bool:
            raise ValueError("knn indices must be integers (got %s)" % idx.dtype)
        idx = idx[:, :K + 1].long()
        if idx.numel() and (int(idx.min()) < -1 or int(idx.max()) >= n):
            raise ValueError("knn entries must lie in [-1, %d)" % n)
        s = torch.sort(idx, 1).values
        if bool(((s[:, 1:] == s[:, :-1]) & (s[:, 1:] >= 0)).any()):
            raise ValueError("a knn row lists the same row twice")
        return _remove_self(idx, K)

    def _build(self, knn):
        n, K, deg, dev = self.x.shape[0], self.build_k, self.degree, self.x.device
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        s = ops._stream()
        ev[0].record()
        knn32 = self._knn(knn)
        ev[1].record()
        fwd = torch.empty((n, deg), dtype=torch.int32, device=dev)
        lib.call("dirb200_graph_prune", ops._ptr(knn32), n, K, deg, ops._ptr(fwd), s)
        ev[2].record()
        # Rev (rule G5): the entries (s, p, t = F(s)[p]) in source order, stably sorted by (t, p)
        t = fwd.view(-1).long()
        ok = t >= 0
        key = (t * deg + torch.arange(deg, device=dev).repeat(n))[ok]
        src = torch.arange(n, device=dev, dtype=torch.int32).repeat_interleave(deg)[ok]
        rev_src = src[torch.sort(key, stable=True).indices].contiguous()
        rev_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(torch.bincount(t[ok], minlength=n), 0, out=rev_off[1:])
        graph = torch.empty((n, deg), dtype=torch.int32, device=dev)
        lib.call("dirb200_graph_merge", ops._ptr(fwd), n, deg, ops._ptr(rev_off), ops._ptr(rev_src), ops._ptr(graph), s)
        ev[3].record()
        torch.cuda.synchronize(dev)
        self.build_ms_ = dict(knn_ms=ev[0].elapsed_time(ev[1]), prune_ms=ev[1].elapsed_time(ev[2]),
                              merge_ms=ev[2].elapsed_time(ev[3]))
        return graph

    def _queries(self, q):
        q = inputs.rows(q, self.x.device, "q")
        if q.shape[1] != self.dim:
            raise ValueError("queries have dimension %d, the index %d" % (q.shape[1], self.dim))
        inputs.check_unit(q, "q")
        pad = self.x.shape[1] - self.dim
        return torch.nn.functional.pad(q, (0, pad)).contiguous() if pad else q

    def _params(self, itopk, width, max_iter, n_seeds):
        itopk = inputs.check_int(itopk, "itopk")
        width = inputs.check_int(width, "width")
        max_iter = inputs.check_int(max_iter, "max_iter", 0)
        n_seeds = inputs.check_int(n_seeds, "n_seeds", 1, self.entry_.shape[0])
        need = smem_bytes(n_seeds, itopk, width, self.degree, max_iter)
        limit = torch.cuda.get_device_properties(self.x.device).shared_memory_per_block_optin
        if need > limit:
            raise ValueError("itopk %d, width %d, max_iter %d, n_seeds %d at degree %d need %d bytes of shared memory per "
                             "query; the device has %d (at most max_iter %d here)"
                             % (itopk, width, max_iter, n_seeds, self.degree, need, limit,
                                max_iter_limit(limit, n_seeds, itopk, width, self.degree)))
        return itopk, width, max_iter, n_seeds

    def seeds(self, q, n_seeds=SEARCH_DEFAULTS["n_seeds"]):
        """Rule G6 -> int64 (Q, n_seeds): each query's best n_seeds rows of the entry sample, in exact order."""
        with torch.cuda.device(self.x.device):
            q = self._queries(q)
            n_seeds = inputs.check_int(n_seeds, "n_seeds", 1, self.entry_.shape[0])
            return self.entry_[self._entry.search(q, n_seeds)[1]]

    def _run(self, q, k, itopk, width, max_iter, n_seeds, visited):
        """Rule G7 for the queries q of _queries (padded like the rows), on the index's device."""
        itopk, width, max_iter, n_seeds = self._params(itopk, width, max_iter, n_seeds)
        k = inputs.check_int(k, "k", 1, itopk)
        dev = q.device
        Q = q.shape[0]
        seeds = self.entry_[self._entry.search(q, n_seeds)[1]].to(torch.int32).contiguous()
        out_s = torch.empty((Q, k), dtype=torch.float64, device=dev)
        out_i = torch.empty((Q, k), dtype=torch.int64, device=dev)
        n_vis = torch.empty(Q, dtype=torch.int32, device=dev)
        n_it = torch.empty(Q, dtype=torch.int32, device=dev)
        vs = vi = None
        if visited:
            cap = n_seeds + max_iter * width * self.degree
            vs = torch.full((Q, cap), -np.inf, dtype=torch.float64, device=dev)
            vi = torch.full((Q, cap), -1, dtype=torch.int64, device=dev)
        lib.call("dirb200_graph_search", ops._ptr(q), Q, q.shape[1], ops._ptr(self.x), self.x.shape[0],
                 ops._ptr(self.graph_), self.degree, ops._ptr(seeds), n_seeds, itopk, width, max_iter, k,
                 ops._ptr(out_s), ops._ptr(out_i), ops._ptr(vi), ops._ptr(vs), ops._ptr(n_vis), ops._ptr(n_it),
                 ops._stream())
        self._stats = dict(queries=Q, visited=n_vis.long(), iterations=n_it.long())
        return out_s, out_i, vs, vi

    def search(self, q, k, itopk=128, width=1, max_iter=256, n_seeds=16):
        """Rule G7 -> (scores fp64 (Q, k), rows int64 (Q, k)): the exact top-k of the rows the traversal visited, padded
        with (-inf, -1); 1 <= k <= itopk.  Parameters whose shared memory exceeds the device's per-block limit are a
        ValueError (at degree 32, itopk 128, width 1 and 16 seeds on an H100, with 227 KB: max_iter up to 511)."""
        with torch.cuda.device(self.x.device):
            return self._run(self._queries(q), k, itopk, width, max_iter, n_seeds, False)[:2]

    def visited(self, q, itopk=128, width=1, max_iter=256, n_seeds=16):
        """Rule G7's visited lists -> (scores fp64, rows int64) (Q, n_seeds + max_iter * width * degree): V(q) in
        arrival order (the seeds in seed order, then each iteration's new rows), padded with (-inf, -1)."""
        with torch.cuda.device(self.x.device):
            return self._run(self._queries(q), 1, itopk, width, max_iter, n_seeds, True)[2:]

    def rank_counts(self, q, t_off, t_rows, t_flags, itopk=128, width=1, max_iter=256, n_seeds=16, exact=None):
        """Rule G8 -> (inside V(q) bool (T,), exact scores fp64 (T,), ranks int64 (T,)) of the targets
        t_rows[t_off[i]:t_off[i+1]] of query i (flagged ones; the others count 0) in the list L_q = V(q) in exact order,
        then every other row in exact order.  a_all comes from exact.rank_counts, exact an ops.Index over the index's
        rows as it holds them (zero-padded to a multiple of 64 columns; built here when not given)."""
        off = np.ascontiguousarray(t_off, dtype=np.int64)
        with torch.cuda.device(self.x.device):
            q = self._queries(q)
            vs, vi = self._run(q, 1, itopk, width, max_iter, n_seeds, True)[2:]
            own = exact is None
            if own:
                exact = ops.Index(self.x)
            try:
                sc, a_all = exact.rank_counts(q, off, t_rows, t_flags)
            finally:
                if own:
                    exact.close()
            return InvertedLists._ranks(off, t_rows, t_flags, sc, a_all, vs, vi)

    def stats(self):
        """The last search: queries, and per query the rows visited |V| and the iterations run (int64 CUDA tensors)."""
        return dict(self._stats)

    def close(self):
        if self._entry is not None:
            self._entry.close()
        self._entry = None
        self.x = self.graph_ = None
