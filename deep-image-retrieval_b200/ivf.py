"""Inverted-file (IVF) search over k-means lists on the GPU (extension; DESIGN.md section 4.10, rules I1-I7).

Rows are bucketed by their exact nearest centre (``cluster.assign``), and each query visits only the ``nprobe`` lists
whose centres score best for it.  The result has an exact definition: the exact top-k of the union R(q) of the probed
lists, in the order of ``ops.Index.search`` (score desc, row asc), with that search's scores.  Probing every list gives
``Index.search`` bit for bit; fewer lists trade recall for speed.  ``tests/ivf_model.py`` restates the rules in numpy.
"""
from __future__ import annotations

import numpy as np
import torch

from . import inputs, ops
from .cluster import SphericalKMeans, assign


class InvertedLists:
    """The k-means lists that IVFIndex and ivfpq.IVFPQIndex share: the centres, the rows of each list and the probe of
    each query (rules I2 and I3)."""

    @staticmethod
    def _centres_of(centres):
        """centres, or the centres of a fitted SphericalKMeans."""
        if isinstance(centres, SphericalKMeans):
            if not hasattr(centres, "cluster_centers_"):
                raise ValueError("the SphericalKMeans has not been fitted")
            return centres.cluster_centers_
        return centres

    def _set_lists(self, labels, c):
        """The lists of rows labelled by their centre (labels int64 (N,), c the (K, D) unit centres): perm_, list_sizes_
        and cell_off_, and the index of the centres that probes them."""
        k = c.shape[0]
        self.perm_ = torch.sort(labels, stable=True).indices
        self.list_sizes_ = torch.bincount(labels, minlength=k)
        self.cell_off_ = torch.zeros(k + 1, dtype=torch.int64, device=labels.device)
        torch.cumsum(self.list_sizes_, 0, out=self.cell_off_[1:])
        self.centres_ = c
        self._centres = ops.Index(c, check_norms=False)

    @property
    def n_lists(self):
        return self.centres_.shape[0]

    def _queries(self, q):
        q = inputs.rows(q, self.centres_.device, "q")
        if q.shape[1] != self.centres_.shape[1]:
            raise ValueError("queries have dimension %d, the index %d" % (q.shape[1], self.centres_.shape[1]))
        inputs.check_unit(q, "q")
        return q

    def _nprobe(self, nprobe):
        return inputs.check_int(nprobe, "nprobe", 1, self.n_lists)

    def probe(self, q, nprobe):
        """Rule I3: the nprobe best lists of each query (score desc, ties to the smaller centre) -> int64 (Q, nprobe)."""
        return self._centres.search(self._queries(q), self._nprobe(nprobe))[1]

    @staticmethod
    def _ranks(off, t_rows, t_flags, sc, a_all, lsc, lix):
        """Rules I7 / P8 from a search of each query's list L_q in exact order (lsc fp64 / lix int64 (Q, depth), tail
        (-inf, -1)) and the exact scores sc and rank counts a_all of the targets (t_rows[off[i]:off[i+1]] of query i)
        -> (inside L_q bool (T,), sc, ranks int64 (T,); 0 for unflagged targets): a target inside L_q ranks after the
        rows of L_q before it, one outside after all of L_q and the rows outside it that rank before it."""
        dev = lix.device
        rows = torch.as_tensor(np.ascontiguousarray(t_rows, dtype=np.int64)).to(dev)
        flags = torch.as_tensor(np.ascontiguousarray(t_flags, dtype=np.uint8)).to(dev)
        t_q = torch.from_numpy(np.repeat(np.arange(lix.shape[0]), np.diff(off))).to(dev)
        a_in = torch.zeros_like(a_all)
        inside = torch.zeros(rows.shape[0], dtype=torch.bool, device=dev)
        step = max(1, (1 << 24) // lix.shape[1])
        for t0 in range(0, rows.shape[0], step):
            tq, tr, ts = t_q[t0:t0 + step], rows[t0:t0 + step], sc[t0:t0 + step]
            ls, li = lsc[tq], lix[tq]
            before = (li >= 0) & ((ls > ts[:, None]) | ((ls == ts[:, None]) & (li < tr[:, None])))
            a_in[t0:t0 + step] = before.sum(1)
            inside[t0:t0 + step] = (li == tr[:, None]).any(1)
        rank = torch.where(inside, a_in, (lix >= 0).sum(1)[t_q] + a_all - a_in)
        return inside, sc, torch.where(flags != 0, rank, torch.zeros_like(rank))

    def close(self):
        self._centres.close()


class IVFIndex(InvertedLists):
    """IVFIndex(X, centres): X (N, D) unit rows (a CUDA tensor, a host array / memmap or a DescriptorStore), centres a
    (K, D) array of unit rows or a fitted SphericalKMeans.

    The build assigns each row to its exact nearest centre (rule I2, ties to the smaller centre), orders the rows stably
    by list and keeps an fp16 copy in that order next to the index's own rows.  labels_ int64 (N,), list_sizes_ int64
    (K,), perm_ (list position -> row) and cell_off_ (K + 1,) are CUDA tensors.  The build is deterministic from (X, C),
    so the centres are all that needs storing."""

    def __init__(self, X, centres, device=None):
        centres = self._centres_of(centres)
        x = inputs.rows(X, device, "X")
        c = inputs.rows(centres, x.device, "centres")
        if x.shape[0] < 1 or c.shape[0] < 1:
            raise ValueError("need at least one row and one centre")
        if x.shape[1] != c.shape[1]:
            raise ValueError("X has dimension %d, the centres %d" % (x.shape[1], c.shape[1]))
        if x.shape[1] % 64:
            raise ValueError("the descriptor dimension must be a multiple of 64 (got %d)" % x.shape[1])
        inputs.check_unit(x, "X")
        inputs.check_unit(c, "centres")
        self.labels_, _ = assign(x, c)
        self._set_lists(self.labels_, c)
        self.index = ops.Index(x)
        self.index.set_lists(self.index.db16[self.perm_].contiguous(), self.perm_, self.cell_off_)

    @classmethod
    def train(cls, X, n_lists, seed=0, max_iter=20, device=None):
        """k-means++ SphericalKMeans with n_lists centres on X, then the lists."""
        x = inputs.rows(X, device, "X")
        km = SphericalKMeans(n_lists, init="k-means++", max_iter=max_iter, seed=seed).fit(x)
        ivf = cls(x, km)
        ivf.kmeans_ = km
        return ivf

    def search(self, q, k, nprobe):
        """Rule I4 -> (scores fp64 (Q, k), rows int64 (Q, k)): the exact top-k of the union of the probed lists."""
        q = self._queries(q)
        k = inputs.check_int(k, "k")
        return self.index.search_lists(q, k, self._centres.search(q, self._nprobe(nprobe))[1])

    def rank_counts(self, q, t_off, t_rows, t_flags, nprobe):
        """Rule I7 -> (inside R(q) bool (T,), exact scores fp64 (T,), ranks int64 (T,)) of the targets t_rows[t_off[i]:t_off[i+1]] of query i
        (flagged ones; the others count 0) in the list L_q = R(q) in exact order, then every other row in exact order.
        a_all comes from Index.rank_counts, L_q from a list search as deep as the largest R(q)."""
        q = self._queries(q)
        nprobe = self._nprobe(nprobe)
        off = np.ascontiguousarray(t_off, dtype=np.int64)
        sc, a_all = self.index.rank_counts(q, off, t_rows, t_flags)
        probes = self._centres.search(q, nprobe)[1]
        depth = max(int(self.list_sizes_[probes].sum(1).max()), 1)
        lsc, lix = self.index.search_lists(q, depth, probes)
        return self._ranks(off, t_rows, t_flags, sc, a_all, lsc, lix)

    def stats(self):
        """Counters (and, with index option 'profile', milliseconds per stage) of the last search."""
        return self.index.lists_stats()

    def set_option(self, key, value):
        self.index.set_option(key, value)

    def close(self):
        self.index.close()
        super().close()
