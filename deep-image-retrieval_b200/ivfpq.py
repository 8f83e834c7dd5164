"""IVF-PQ: inverted lists of product-quantisation codes, with exact re-ranking (extension; DESIGN.md section 4.11,
rules P1-P8).

The lists are those of ``ivf.IVFIndex`` (rule I2).  Each row is stored as M one-byte codes of its residual to its list
centre; a query scores the rows of its probed lists by table lookups (the ADC score, rule P5), keeps the best R of
them (rule P6) and re-ranks those exactly against the fp32 rows (rule P7).  The rows need not be on the device: with
``rows="host"`` they stay in pinned host memory and only the candidates cross the bus.  With R at least the number of
probed rows the result is ``IVFIndex.search`` bit for bit.  ``tests/ivfpq_model.py`` restates the rules in numpy.
"""
from __future__ import annotations

import numpy as np
import torch

from . import inputs, lib, ops
from .cluster import SphericalKMeans, assign
from .ivf import InvertedLists

MS = (8, 16, 32, 64, 128)       # rule P2
MAX_SUB = 256                   # the kernels' largest sub-vector D / M
TRAIN_SIZE = 65536              # rule P3's default training set (at most N rows)
RANK_REFINE = 400               # rank_counts' default R: 4k at k = 100
MAX_QUERIES = 65535             # queries per dirb200_pq_search


def _i(v):
    return int(v.item()) if isinstance(v, torch.Tensor) else int(v)


def _plan(n, chunk_rows, train_rows):
    """The build's chunks [(a, b, lo, hi)]: rows [a, b) in order, and train_rows[lo:hi] (sorted) the training rows
    among them."""
    out = []
    for a in range(0, n, chunk_rows):
        b = min(n, a + chunk_rows)
        lo, hi = np.searchsorted(train_rows, [a, b])
        out.append((a, b, int(lo), int(hi)))
    return out


def _check_shape(d, M):
    if isinstance(M, bool) or not isinstance(M, (int, np.integer)) or M not in MS:
        raise ValueError("M must be one of %s (got %r)" % (MS, M))
    if d % 64:
        raise ValueError("the descriptor dimension must be a multiple of 64 (got %d)" % d)
    if d % M:
        raise ValueError("M = %d does not divide the dimension %d" % (M, d))
    if d // M > MAX_SUB:
        raise ValueError("sub-vectors of %d dimensions: at most %d (use a larger M)" % (d // M, MAX_SUB))
    return int(M)


class IVFPQIndex(InvertedLists):
    """IVFPQIndex(X, centres, M): X (N, D) unit rows (a CUDA tensor, a host array / memmap or a DescriptorStore),
    centres a (K, D) array of unit rows or a fitted SphericalKMeans, M codes per row (rule P2).

    train_size: rows of the codebook training set (rule P3; default min(N, 65536)), pq_iter: Lloyd iterations,
    seed: numpy.random.default_rng seed of the training rows and the initial codewords.  rows: "device" keeps the fp32
    rows on the device for the refinement, "host" keeps a pinned host copy read in place (only the candidates cross
    the bus).  The build reads X in chunks of chunk_rows rows, so with rows="host" the device never holds all of them.

    After the build: codebooks_ (M, 256, D / M) fp32, codes_ (N, M) uint8 in list order, perm_ (list position -> row),
    list_sizes_ (K,), cell_off_ (K + 1,) (CUDA tensors), device_bytes_ and empty_codewords_ (codewords kept by the last
    update because no training row chose them)."""

    def __init__(self, X, centres, M, train_size=None, pq_iter=25, seed=0, rows="device", chunk_rows=1 << 16,
                 device=None):
        centres = self._centres_of(centres)
        if rows not in ("device", "host"):
            raise ValueError("rows must be 'device' or 'host' (got %r)" % (rows,))
        dev = inputs.device(device, X)
        src = inputs.Rows(X)
        n, d = src.n, src.d
        c = inputs.rows(centres, dev, "centres")
        if n < 1 or c.shape[0] < 1:
            raise ValueError("need at least one row and one centre")
        if n >= 1 << 31:
            raise ValueError("at most 2^31 - 1 rows (got %d)" % n)
        if c.shape[1] != d:
            raise ValueError("X has dimension %d, the centres %d" % (d, c.shape[1]))
        self.M = _check_shape(d, M)
        chunk_rows = inputs.check_int(chunk_rows, "chunk_rows")
        pq_iter = int(pq_iter)
        if pq_iter < 0:
            raise ValueError("pq_iter must be >= 0 (got %d)" % pq_iter)
        T = min(n, TRAIN_SIZE) if train_size is None else inputs.check_int(train_size, "train_size", 1, n)
        if T < 256:
            raise ValueError("the codebooks need at least 256 training rows (got %d)" % T)
        inputs.check_unit(c, "centres")
        rng = np.random.default_rng(seed)
        train_rows = np.sort(rng.choice(n, T, replace=False))
        init = rng.choice(T, 256, replace=False)

        # pass 1: labels (rule P1), the training rows and the kept rows, chunk by chunk
        labels = torch.empty(n, dtype=torch.int64, device=dev)
        xt = torch.empty((T, d), dtype=torch.float32, device=dev)
        whole = isinstance(X, torch.Tensor) and X.is_cuda and X.dtype == torch.float32 and X.is_contiguous() \
            and X.device == dev
        if rows == "host":
            self.rows_ = torch.empty((n, d), dtype=torch.float32, pin_memory=True)
        else:
            self.rows_ = X if whole else torch.empty((n, d), dtype=torch.float32, device=dev)
        plan = _plan(n, chunk_rows, train_rows)
        self.chunks_ = len(plan)
        for a, b, lo, hi in plan:
            xc = src.get(a, b, dev)
            inputs.check_unit(xc, "X")
            labels[a:b] = assign(xc, c)[0]
            if hi > lo:
                xt[lo:hi] = xc[torch.from_numpy(train_rows[lo:hi] - a).to(dev)]
            if self.rows_ is not X:
                self.rows_[a:b].copy_(xc)
        self._set_lists(labels, c)

        # rule P3: codebooks from the residuals of the training rows
        lt = labels[torch.from_numpy(train_rows).to(dev)].contiguous()
        sub = d // self.M
        i0 = torch.from_numpy(init).to(dev)
        res0 = xt[i0] - c[lt[i0]]                               # fl32(x - c), elementwise
        self.codebooks_ = res0.view(256, self.M, sub).permute(1, 0, 2).contiguous()
        codes_t = torch.empty((self.M, T), dtype=torch.uint8, device=dev)
        empty = torch.zeros(1, dtype=torch.int64, device=dev)
        s = ops._stream()
        for _ in range(pq_iter):
            lib.call("dirb200_pq_assign", ops._ptr(xt), T, d, ops._ptr(lt), ops._ptr(c), ops._ptr(self.codebooks_),
                     self.M, ops._ptr(codes_t), 1, s)
            lib.call("dirb200_pq_update", ops._ptr(xt), T, d, ops._ptr(lt), ops._ptr(c), ops._ptr(codes_t), self.M,
                     ops._ptr(self.codebooks_), ops._ptr(empty), s)
        self.empty_codewords_ = _i(empty)
        del xt, codes_t

        # rule P4: the codes, chunk by chunk, then in list order
        codes = torch.empty((n, self.M), dtype=torch.uint8, device=dev)
        for a, b, _, _ in plan:
            xc = X[a:b] if whole else self.rows_[a:b].to(dev, non_blocking=True)
            lib.call("dirb200_pq_assign", ops._ptr(xc), b - a, d, ops._ptr(labels[a:b]), ops._ptr(c),
                     ops._ptr(self.codebooks_), self.M, ops._ptr(codes[a:b]), 0, s)
        self.codes_ = codes[self.perm_].contiguous()
        del codes, labels
        self.rows = rows
        self.ws_budget = 1 << 30
        self.profile = False
        self._stats = {}
        held = [self.codes_, self.perm_, self.list_sizes_, self.cell_off_, self.centres_, self.codebooks_,
                self._centres.db32, self._centres.db16] + ([self.rows_] if rows == "device" else [])
        self.device_bytes_ = sum(t.numel() * t.element_size() for t in held)

    @classmethod
    def train(cls, X, n_lists, M, seed=0, max_iter=20, fit_rows=None, device=None, **kw):
        """k-means++ SphericalKMeans with n_lists centres (seed, max_iter), then the index (kw: the constructor's).
        The lists are fitted on the device: on every row when X is a CUDA tensor or has at most fit_rows rows (default:
        as many as a quarter of the free device memory holds), else on fit_rows rows drawn without replacement by
        numpy.random.default_rng(seed) (sorted)."""
        dev = inputs.device(device, X)
        src = inputs.Rows(X)
        if fit_rows is None:
            fit_rows = max(n_lists, torch.cuda.mem_get_info(dev)[0] // (4 * 4 * src.d))
        if isinstance(X, torch.Tensor) and X.is_cuda or src.n <= fit_rows:
            xf = src.get(0, src.n, dev)
        else:
            sel = np.sort(np.random.default_rng(seed).choice(src.n, int(fit_rows), replace=False))
            xf = torch.empty((len(sel), src.d), dtype=torch.float32, device=dev)
            for a, b, lo, hi in _plan(src.n, 1 << 16, sel):
                if hi > lo:
                    xf[lo:hi] = src.get(a, b, dev)[torch.from_numpy(sel[lo:hi] - a).to(dev)]
        km = SphericalKMeans(n_lists, init="k-means++", max_iter=max_iter, seed=seed).fit(xf)
        del xf
        index = cls(X, km, M, seed=seed, device=dev, **kw)
        index.kmeans_ = km
        return index

    def search(self, q, k, nprobe, refine=None):
        """Rules P5-P7 -> (scores fp64 (Q, k), rows int64 (Q, k)): the exact top-k of the best refine (R, default 4k)
        probed rows by ADC score, padded with (-inf, -1)."""
        q = self._queries(q)
        k = inputs.check_int(k, "k")
        R = 4 * k if refine is None else inputs.check_int(refine, "refine", k)
        nprobe = self._nprobe(nprobe)
        R = max(k, min(R, self.perm_.shape[0]))       # C_q never holds more than N rows
        dev = q.device
        Q, d = q.shape
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)] if self.profile else None
        psc, probes = self._centres.search(q, nprobe)
        r_size = self.list_sizes_[probes].sum(1)
        cum = np.concatenate([[0], np.cumsum(r_size.cpu().numpy())])
        out_s = torch.empty((Q, k), dtype=torch.float64, device=dev)
        out_i = torch.empty((Q, k), dtype=torch.int64, device=dev)
        ms = (lib.f64 * 3)() if self.profile else None
        st = dict(queries=Q, blocks=0, segments=Q * nprobe, rows_scanned=int(cum[-1]),
                  candidates=int(np.minimum(np.diff(cum), R).sum()))
        if self.profile:
            st.update(tables_ms=0.0, scan_ms=0.0, select_ms=0.0, refine_ms=0.0)
        s = ops._stream()
        q0 = 0
        while q0 < Q:
            qb = min(Q - q0, MAX_QUERIES)
            while True:
                total = int(cum[q0 + qb] - cum[q0])
                need = lib.raw("dirb200_pq_search_ws_bytes")(qb, total, R) + qb * self.M * 1024
                if need <= self.ws_budget or qb == 1:
                    break
                qb = (qb + 1) // 2
            qq = q[q0:q0 + qb]
            qoff = torch.from_numpy(cum[q0:q0 + qb + 1] - cum[q0]).to(dev)
            tables = torch.empty((qb, self.M, 256), dtype=torch.float32, device=dev)
            ws = ops.workspace(lib.raw("dirb200_pq_search_ws_bytes")(qb, total, R), dev)
            if ev:
                ev[0].record()
            lib.call("dirb200_pq_tables", ops._ptr(qq), qb, d, ops._ptr(self.codebooks_), self.M, ops._ptr(tables), s)
            if ev:
                ev[1].record()
            lib.call("dirb200_pq_search", ops._ptr(qq), qb, d, ops._ptr(tables), self.M,
                     ops._ptr(probes[q0:q0 + qb]), ops._ptr(psc[q0:q0 + qb]), nprobe, ops._ptr(self.codes_),
                     ops._ptr(self.perm_), ops._ptr(self.cell_off_), ops._ptr(qoff), total,
                     ops._ptr(self.rows_), R, k, ops._ptr(ws), ops._ptr(out_s[q0:q0 + qb]),
                     ops._ptr(out_i[q0:q0 + qb]), None if ms is None else lib.C.cast(ms, lib.C.c_void_p), s)
            if ms is not None:
                st["tables_ms"] += ev[0].elapsed_time(ev[1])
                st["scan_ms"] += ms[0]
                st["select_ms"] += ms[1]
                st["refine_ms"] += ms[2]
            st["blocks"] += 1
            q0 += qb
        self._stats = st
        return out_s, out_i

    def rank_counts(self, q, t_off, t_rows, t_flags, nprobe, refine=None, exact=None):
        """Rule P8 -> (inside C_q bool (T,), exact scores fp64 (T,), ranks int64 (T,)) of the targets
        t_rows[t_off[i]:t_off[i+1]] of query i (flagged ones; the others count 0) in the list L_q = C_q in exact order,
        then every other row in exact order.  refine: R (default 400).  a_all comes from exact.rank_counts, exact an
        ops.Index over the same rows (built here from the kept rows when not given), a_in from a search as deep as the
        largest C_q."""
        q = self._queries(q)
        nprobe = self._nprobe(nprobe)
        R = RANK_REFINE if refine is None else inputs.check_int(refine, "refine")
        off = np.ascontiguousarray(t_off, dtype=np.int64)
        own = exact is None
        if own:
            exact = ops.Index(self.rows_.to(q.device))
        try:
            sc, a_all = exact.rank_counts(q, off, t_rows, t_flags)
        finally:
            if own:
                exact.close()
        depth = max(1, min(R, int(self.list_sizes_[self._centres.search(q, nprobe)[1]].sum(1).max())))
        lsc, lix = self.search(q, depth, nprobe, refine=max(R, depth))
        return self._ranks(off, t_rows, t_flags, sc, a_all, lsc, lix)

    def stats(self):
        """The last search: queries, query blocks, (query, probe) segments, rows scanned, candidates refined, and with
        set_option('profile', 1) the milliseconds of the tables, the scan, the selection and the refinement."""
        return dict(self._stats)

    def set_option(self, key, value):
        """'ws_budget': bytes of workspace per query block (tables included; default 1 GiB); 'profile': 0 / 1."""
        if key == "ws_budget":
            self.ws_budget = int(value)
        elif key == "profile":
            self.profile = bool(value)
        else:
            raise ValueError("unknown option %r (ws_budget, profile)" % (key,))

    def close(self):
        super().close()
        for name in ("codes_", "perm_", "rows_", "codebooks_"):
            setattr(self, name, None)
