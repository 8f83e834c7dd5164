"""Diffusion re-ranking on the GPU (extension; Zhou et al., "Ranking on Data Manifolds", NIPS 2003; Iscen et al.,
"Efficient Diffusion on Region Manifolds", CVPR 2017).

The database rows are linked by an exact mutual-kNN graph, normalised to S = D^-1/2 A D^-1/2; a query's scores are
the solution f of (I - alpha S) f = y, y holding the query's top-kq scores raised to gamma, solved by conjugate
gradient in fp64.  Rows are then ranked by f (descending, ties -> lower index).  The rules are stated in DESIGN.md
section 4.7; every step runs on the kernels of csrc/diffusion.cu and the exact search of ops.Index.

    d = Diffusion(bdescs)                     # graph of the database (device or host rows, unit norm)
    f, iters, resid = d.solve(qdescs)         # (Q, N) scores
    scores, idx = d.search(qdescs, 100)       # (Q, 100) ranking lists
    scores, above = d.rank_counts(qdescs, t_off, t_rows, t_flags)

Truncation (Iscen et al. 2017; DESIGN.md section 4.7, rules T1-T6): each query is solved on the subgraph of its own
m nearest rows R_q only, renormalised, and every other row is ranked after R_q in exact-score order.

    d = Diffusion(bdescs, truncation=True)    # also keeps A and u of the graph
    rows, f, iters, resid = d.solve_truncated(qdescs, 1000)
    scores, idx = d.search(qdescs, 100, truncate=1000)
    inside, value, above = d.rank_counts_truncated(qdescs, t_off, t_rows, t_flags, 1000)
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np
import torch

from . import lib, ops
from .inputs import rows64

# Iscen et al. 2017, experiments on global descriptors (see DESIGN.md section 4.7): k = 50 mutual neighbours, the
# kq = 10 nearest rows seed a query, gamma = 3, alpha = 0.99, 20 conjugate-gradient iterations.  tol = 0 keeps the
# paper's fixed iteration count.
DEFAULTS = dict(k=50, kq=10, gamma=3.0, alpha=0.99, iters=20, tol=0.0)
WS_BUDGET = 4 << 30           # bytes of the solver's per-block arrays (five N x Qb fp64 arrays)
MAX_Q_BLOCK = 65535           # queries per kernel call (the rank-count and top-k grids take one row per query)


def check_params(k=None, kq=None, gamma=None, alpha=None, iters=None, tol=None):
    """ValueError for a parameter outside its range (None = not given)."""
    if k is not None and not (int(k) == k and k >= 1):
        raise ValueError("diffusion: k must be an integer >= 1 (got %r)" % (k,))
    if kq is not None and not (int(kq) == kq and kq >= 1):
        raise ValueError("diffusion: kq must be an integer >= 1 (got %r)" % (kq,))
    if gamma is not None and not gamma > 0:
        raise ValueError("diffusion: gamma must be > 0 (got %r)" % (gamma,))
    if alpha is not None and not 0 <= alpha < 1:
        raise ValueError("diffusion: alpha must satisfy 0 <= alpha < 1 (got %r)" % (alpha,))
    if iters is not None and not (int(iters) == iters and iters >= 1):
        raise ValueError("diffusion: iters must be an integer >= 1 (got %r)" % (iters,))
    if tol is not None and not tol >= 0:
        raise ValueError("diffusion: tol must be >= 0 (got %r)" % (tol,))


def check_truncate(m):
    """ValueError unless m (the truncation depth) is an integer >= 1."""
    if isinstance(m, bool) or not (float(m) == int(m) and m >= 1):
        raise ValueError("diffusion: the truncation depth m must be an integer >= 1 (got %r)" % (m,))
    return int(m)


class Graph(NamedTuple):
    """CSR of S: row_ptr int64 (N+1,), col int32 (nnz,) ascending within a row, val fp64 (nnz,)."""
    row_ptr: torch.Tensor
    col: torch.Tensor
    val: torch.Tensor


class Weights(NamedTuple):
    """The graph before normalisation, on the CSR of Graph: a fp64 (nnz,) = A_ij, u fp64 (N,) = 1/sqrt(d_i)."""
    a: torch.Tensor
    u: torch.Tensor


def graph_from_knn(idx, scores, k, gamma, weights=False):
    """The CSR of S from the exact top-(k+1) lists of the database against itself: idx int64 / scores fp64 (N, width)
    CUDA tensors, width <= k + 1, entries in [0, N) or -1 (dirb200_diffusion_graph).  weights=True -> (Graph, Weights)
    from dirb200_diffusion_graph_weights (the same Graph bits)."""
    check_params(k=k, gamma=gamma)
    ops._chk(idx, torch.int64, "idx")
    ops._chk(scores, torch.float64, "scores")
    if idx.dim() != 2 or tuple(scores.shape) != tuple(idx.shape) or not 1 <= idx.shape[1] <= int(k) + 1:
        raise ValueError("diffusion: idx and scores must be (N, width) with 1 <= width <= k + 1 = %d" % (int(k) + 1))
    if idx.numel() and not (int(idx.min()) >= -1 and int(idx.max()) < idx.shape[0]):
        raise ValueError("diffusion: neighbour indices must lie in [0, %d) or be -1" % idx.shape[0])
    n, width = idx.shape
    dev = idx.device
    ws = ops.workspace(lib.raw("dirb200_diffusion_graph_workspace_bytes")(n, int(k)), dev)
    row_ptr = torch.empty(n + 1, dtype=torch.int64, device=dev)
    col = torch.empty(n * int(k), dtype=torch.int32, device=dev)
    val = torch.empty(n * int(k), dtype=torch.float64, device=dev)
    if weights:
        a = torch.empty(n * int(k), dtype=torch.float64, device=dev)
        u = torch.empty(n, dtype=torch.float64, device=dev)
        lib.call("dirb200_diffusion_graph_weights", ops._ptr(idx), ops._ptr(scores), n, width, int(k), float(gamma),
                 ops._ptr(ws), ops._ptr(row_ptr), ops._ptr(col), ops._ptr(val), ops._ptr(a), ops._ptr(u), ops._stream())
        nnz = int(row_ptr[-1])
        return Graph(row_ptr, col[:nnz].clone(), val[:nnz].clone()), Weights(a[:nnz].clone(), u)
    lib.call("dirb200_diffusion_graph", ops._ptr(idx), ops._ptr(scores), n, width, int(k), float(gamma), ops._ptr(ws),
             ops._ptr(row_ptr), ops._ptr(col), ops._ptr(val), ops._stream())
    nnz = int(row_ptr[-1])
    return Graph(row_ptr, col[:nnz].clone(), val[:nnz].clone())


class Local(NamedTuple):
    """The subgraphs of a block of Qb queries (dirb200_diffusion_trunc_build), m' local rows each: rows int64 (Qb, m')
    ascending, cnt int32 (Qb, m'), col int32 / val fp64 (Qb, kw, m') ELL column-major (val = S'), d / u / y fp64
    (Qb, m') = d', u', y'."""
    rows: torch.Tensor
    cnt: torch.Tensor
    col: torch.Tensor
    val: torch.Tensor
    d: torch.Tensor
    u: torch.Tensor
    y: torch.Tensor


class Diffusion:
    """Diffusion over the mutual-kNN graph of the database rows `bdescs` ((N, D) fp32, unit norm; CUDA tensor or host
    array).  `graph` holds the CSR of S as CUDA tensors; with truncation=True, `weights` also holds A and u (the
    subgraphs of truncated diffusion are renormalised from A), else None."""

    def __init__(self, bdescs, k=DEFAULTS["k"], gamma=DEFAULTS["gamma"], ws_budget=WS_BUDGET, knn=None,
                 truncation=False):
        """knn: optional (scores, idx) = self.index.search(rows, k + 1) when the caller already has those lists.
        truncation: keep A and u for solve_truncated / search(truncate=m) / rank_counts_truncated (nnz x 8 bytes)."""
        check_params(k=k, gamma=gamma)
        self.k, self.gamma, self.ws_budget = int(k), float(gamma), int(ws_budget)
        self.dim = bdescs.shape[1]
        self.db = rows64(bdescs)
        self.n = self.db.shape[0]
        if self.n < 1:
            raise ValueError("diffusion: the database is empty")
        self.index = ops.Index(self.db)
        sc, idx = self.index.search(self.db, self.k + 1) if knn is None else knn
        if truncation:
            self.graph, self.weights = graph_from_knn(idx, sc, self.k, self.gamma, weights=True)
            self.ell = max(1, int((self.graph.row_ptr[1:] - self.graph.row_ptr[:-1]).max()))   # longest row
        else:
            self.graph = graph_from_knn(idx, sc, self.k, self.gamma)
            self.weights = None

    def query_block(self, nq):
        """Queries per solve block: the solver holds about five N x Qb fp64 arrays within ws_budget."""
        return int(max(1, min(nq, self.ws_budget // (5 * 8 * self.n))))

    def _blocks(self, qdescs, kq, alpha, iters, tol, q_block):
        """Yields (q0, f [N][Qb] fp64, iters (Qb,) int32, resid (Qb,) fp64) per block of queries."""
        check_params(kq=kq, alpha=alpha, iters=iters, tol=tol)
        if qdescs.shape[1] != self.dim:
            raise ValueError("diffusion: query dimension %d differs from the database's %d" % (qdescs.shape[1], self.dim))
        q = rows64(qdescs)
        nq, n = q.shape[0], self.n
        qb = min(int(q_block) if q_block else self.query_block(nq), MAX_Q_BLOCK)
        g = self.graph
        dev = q.device
        for q0 in range(0, nq, qb):
            qc = q[q0:q0 + qb].contiguous()
            b = qc.shape[0]
            sc, idx = self.index.search(qc, int(kq))
            y = torch.empty((n, b), dtype=torch.float64, device=dev)
            lib.call("dirb200_diffusion_seeds", ops._ptr(idx), ops._ptr(sc), b, int(kq), self.gamma, n, ops._ptr(y),
                     ops._stream())
            ws = ops.workspace(lib.raw("dirb200_diffusion_solve_workspace_bytes")(n, b), dev)
            f = torch.empty((n, b), dtype=torch.float64, device=dev)
            it = torch.empty(b, dtype=torch.int32, device=dev)
            res = torch.empty(b, dtype=torch.float64, device=dev)
            lib.call("dirb200_diffusion_solve", ops._ptr(g.row_ptr), ops._ptr(g.col), ops._ptr(g.val), n, ops._ptr(y), b,
                     float(alpha), int(iters), float(tol), ops._ptr(ws), ops._ptr(f), ops._ptr(it), ops._ptr(res),
                     ops._stream())
            del ws, y
            yield q0, f, it, res

    def solve(self, qdescs, kq=DEFAULTS["kq"], alpha=DEFAULTS["alpha"], iters=DEFAULTS["iters"], tol=DEFAULTS["tol"],
              q_block=None):
        """-> (f fp64 (Q, N), iterations int32 (Q,), final recurrence residual ||r|| fp64 (Q,)), CUDA tensors.
        q_block: queries per solve (default: from ws_budget); the result does not depend on it."""
        nq = qdescs.shape[0]
        f = torch.empty((nq, self.n), dtype=torch.float64, device="cuda")
        its = torch.empty(nq, dtype=torch.int32, device="cuda")
        res = torch.empty(nq, dtype=torch.float64, device="cuda")
        for q0, fb, it, r in self._blocks(qdescs, kq, alpha, iters, tol, q_block):
            b = fb.shape[1]
            f[q0:q0 + b] = fb.t()
            its[q0:q0 + b] = it
            res[q0:q0 + b] = r
        return f, its, res

    def search(self, qdescs, k, kq=DEFAULTS["kq"], alpha=DEFAULTS["alpha"], iters=DEFAULTS["iters"],
               tol=DEFAULTS["tol"], q_block=None, truncate=None):
        """Exact top-k of each query's f (f descending, ties -> lower index, -0 == +0; dirb200_diffusion_topk), any
        1 <= k <= N -> (f scores fp64 (Q, k), rows int64 (Q, k)), CUDA tensors.
        truncate=m: rule T6 instead - the m' = min(m, N) rows of R_q by f' (the same order), then the other rows in
        exact-score order; scores hold f' for the first m' entries and the exact score after them."""
        if not (int(k) == k and 1 <= k <= self.n):
            raise ValueError("diffusion: k must be an integer in [1, %d] (got %r)" % (self.n, k))
        k = int(k)
        if truncate is not None:
            return self._search_truncated(qdescs, k, truncate, kq, alpha, iters, tol, q_block)
        nq = qdescs.shape[0]
        scores = torch.empty((nq, k), dtype=torch.float64, device="cuda")
        idx = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        for q0, fb, _, _ in self._blocks(qdescs, kq, alpha, iters, tol, q_block):
            b = fb.shape[1]
            ws = ops.workspace(lib.raw("dirb200_diffusion_topk_workspace_bytes")(b, k), fb.device)
            lib.call("dirb200_diffusion_topk", ops._ptr(fb), self.n, b, k, ops._ptr(ws), ops._ptr(scores[q0:q0 + b]),
                     ops._ptr(idx[q0:q0 + b]), ops._stream())
        return scores, idx

    def _targets(self, nq, t_off, t_rows, t_flags):
        """The targets of nq queries (host CSR) -> (off int64 (nq+1,), rows int64 (T,), flags uint8 (T,)), checked."""
        off = np.ascontiguousarray(t_off, dtype=np.int64)
        rows = np.ascontiguousarray(t_rows, dtype=np.int64)
        flags = np.ascontiguousarray(t_flags, dtype=np.uint8)
        if off.shape != (nq + 1,) or off[0] != 0 or off[-1] != rows.shape[0] or np.any(np.diff(off) < 0):
            raise ValueError("diffusion: t_off must be non-decreasing offsets from 0 to len(t_rows), one per query + 1")
        if flags.shape != rows.shape:
            raise ValueError("diffusion: t_flags must have the shape of t_rows")
        if rows.size and (rows.min() < 0 or rows.max() >= self.n):
            raise ValueError("diffusion: target rows must lie in [0, %d)" % self.n)
        return off, rows, flags

    def rank_counts(self, qdescs, t_off, t_rows, t_flags, kq=DEFAULTS["kq"], alpha=DEFAULTS["alpha"],
                    iters=DEFAULTS["iters"], tol=DEFAULTS["tol"], q_block=None):
        """For the targets of each query (host CSR: t_off int (Q+1,), t_rows int64 (T,), t_flags uint8 (T,)) ->
        (f at each target fp64 (T,), rows ranking before each flagged target int64 (T,); 0 when unflagged), CUDA
        tensors: the contract of ops.Index.rank_counts with f in place of the exact score."""
        off, rows, flags = self._targets(qdescs.shape[0], t_off, t_rows, t_flags)
        T = rows.shape[0]
        scores = torch.zeros(T, dtype=torch.float64, device="cuda")
        above = torch.zeros(T, dtype=torch.int64, device="cuda")
        for q0, fb, _, _ in self._blocks(qdescs, kq, alpha, iters, tol, q_block):
            b = fb.shape[1]
            lo, hi = int(off[q0]), int(off[q0 + b])
            if hi == lo:
                continue
            o = np.ascontiguousarray(off[q0:q0 + b + 1] - lo, dtype=np.int32)
            o_d = torch.from_numpy(o).to(fb.device)
            r_d = torch.from_numpy(rows[lo:hi]).to(fb.device)
            f_d = torch.from_numpy(flags[lo:hi]).to(fb.device)
            ws = ops.workspace(lib.raw("dirb200_diffusion_rank_count_workspace_bytes")(b, hi - lo), fb.device)
            lib.call("dirb200_diffusion_rank_count", ops._ptr(fb), self.n, b, o.ctypes.data_as(C.c_void_p), ops._ptr(o_d),
                     ops._ptr(r_d), ops._ptr(f_d), hi - lo, ops._ptr(ws), ops._ptr(scores[lo:hi]), ops._ptr(above[lo:hi]),
                     ops._stream())
        return scores, above

    # ------------------------------------------------------------------------------------------------ truncation
    def trunc_query_block(self, nq, m, depth=0):
        """Queries per truncated block: the subgraphs (ELL of kw entries per local row), the vectors, the exact lists
        to `depth` and the sort workspaces of the m' local rows stay within ws_budget."""
        kw = self.ell
        p2 = 1 << max(0, (m - 1).bit_length())
        per_q = m * (12 * kw + 4 + 8 * 7 + 32 + 20) + 16 * max(depth, m) + 8 * p2 + 16 * 2048
        return int(max(1, min(nq, self.ws_budget // per_q, MAX_Q_BLOCK)))

    def _trunc_blocks(self, qdescs, m, kq, alpha, iters, tol, q_block, depth=0):
        """Yields (q0, list scores (Qb, depth') fp64, list idx int64, Local, f' (Qb, m'), iters, resid) per block;
        depth' = max(depth, m') entries of each query's exact list, m' = min(m, N)."""
        if self.weights is None:
            raise ValueError("diffusion: truncation needs the graph's weights: build with Diffusion(..., truncation=True)")
        m = min(check_truncate(m), self.n)
        check_params(kq=kq, alpha=alpha, iters=iters, tol=tol)
        if int(kq) > m:
            raise ValueError("diffusion: kq = %d exceeds the truncation depth m' = min(m, N) = %d" % (kq, m))
        if qdescs.shape[1] != self.dim:
            raise ValueError("diffusion: query dimension %d differs from the database's %d" % (qdescs.shape[1], self.dim))
        q = rows64(qdescs)
        nq, n, kw = q.shape[0], self.n, self.ell
        depth = max(int(depth), m)
        qb = min(int(q_block) if q_block else self.trunc_query_block(nq, m, depth), MAX_Q_BLOCK)
        g, w = self.graph, self.weights
        dev = q.device
        for q0 in range(0, nq, qb):
            qc = q[q0:q0 + qb].contiguous()
            b = qc.shape[0]
            sc, idx = self.index.search(qc, depth)
            li, ls = (idx, sc) if depth == m else (idx[:, :m].contiguous(), sc[:, :m].contiguous())
            loc = Local(torch.empty((b, m), dtype=torch.int64, device=dev), torch.empty((b, m), dtype=torch.int32, device=dev),
                        torch.empty((b, kw, m), dtype=torch.int32, device=dev),
                        torch.empty((b, kw, m), dtype=torch.float64, device=dev),
                        *(torch.empty((b, m), dtype=torch.float64, device=dev) for _ in range(3)))
            ws = ops.workspace(lib.raw("dirb200_diffusion_trunc_build_workspace_bytes")(b, m), dev)
            lib.call("dirb200_diffusion_trunc_build", ops._ptr(g.row_ptr), ops._ptr(g.col), ops._ptr(w.a), n, kw,
                     ops._ptr(li), ops._ptr(ls), b, m, int(kq), self.gamma, ops._ptr(ws), *(ops._ptr(t) for t in loc),
                     ops._stream())
            ws = ops.workspace(lib.raw("dirb200_diffusion_trunc_solve_workspace_bytes")(b, m), dev)
            f = torch.empty((b, m), dtype=torch.float64, device=dev)
            it = torch.empty(b, dtype=torch.int32, device=dev)
            res = torch.empty(b, dtype=torch.float64, device=dev)
            lib.call("dirb200_diffusion_trunc_solve", ops._ptr(loc.cnt), ops._ptr(loc.col), ops._ptr(loc.val), kw,
                     ops._ptr(loc.y), b, m, float(alpha), int(iters), float(tol), ops._ptr(ws), ops._ptr(f), ops._ptr(it),
                     ops._ptr(res), ops._stream())
            del ws
            yield q0, sc, idx, loc, f, it, res

    def subgraphs(self, qdescs, m, kq=DEFAULTS["kq"], q_block=None):
        """The local systems of truncated diffusion (rules T1-T4) for all queries in one block -> Local."""
        nq = qdescs.shape[0]
        for _, _, _, loc, _, _, _ in self._trunc_blocks(qdescs, m, kq, DEFAULTS["alpha"], 1, 0.0, q_block or nq):
            return loc

    def solve_truncated(self, qdescs, m, kq=DEFAULTS["kq"], alpha=DEFAULTS["alpha"], iters=DEFAULTS["iters"],
                        tol=DEFAULTS["tol"], q_block=None):
        """Rules T1-T5 -> (local rows int64 (Q, m') ascending, f' fp64 (Q, m'), iterations int32 (Q,), final recurrence
        residual fp64 (Q,)), CUDA tensors, m' = min(m, N).  With m >= N this is solve()'s result bit for bit.
        q_block: queries per block (default: from ws_budget); the result does not depend on it."""
        nq = qdescs.shape[0]
        mm = min(check_truncate(m), self.n)
        rows = torch.empty((nq, mm), dtype=torch.int64, device="cuda")
        f = torch.empty((nq, mm), dtype=torch.float64, device="cuda")
        its = torch.empty(nq, dtype=torch.int32, device="cuda")
        res = torch.empty(nq, dtype=torch.float64, device="cuda")
        for q0, _, _, loc, fb, it, r in self._trunc_blocks(qdescs, m, kq, alpha, iters, tol, q_block):
            b = fb.shape[0]
            rows[q0:q0 + b] = loc.rows
            f[q0:q0 + b] = fb
            its[q0:q0 + b] = it
            res[q0:q0 + b] = r
        return rows, f, its, res

    def _search_truncated(self, qdescs, k, m, kq, alpha, iters, tol, q_block):
        nq = qdescs.shape[0]
        scores = torch.empty((nq, k), dtype=torch.float64, device="cuda")
        idx = torch.empty((nq, k), dtype=torch.int64, device="cuda")
        for q0, ls, li, loc, fb, _, _ in self._trunc_blocks(qdescs, m, kq, alpha, iters, tol, q_block, depth=k):
            b, mm = fb.shape
            ws = ops.workspace(lib.raw("dirb200_diffusion_trunc_topk_workspace_bytes")(b, mm, k), fb.device)
            lib.call("dirb200_diffusion_trunc_topk", ops._ptr(loc.rows), ops._ptr(fb), b, mm, ops._ptr(li), ops._ptr(ls),
                     li.shape[1], k, ops._ptr(ws), ops._ptr(scores[q0:q0 + b]), ops._ptr(idx[q0:q0 + b]), ops._stream())
        return scores, idx

    def rank_counts_truncated(self, qdescs, t_off, t_rows, t_flags, m, kq=DEFAULTS["kq"], alpha=DEFAULTS["alpha"],
                              iters=DEFAULTS["iters"], tol=DEFAULTS["tol"], q_block=None):
        """Rule T6 for the targets of each query (host CSR as in rank_counts) -> (inside bool (T,): the row lies in
        R_q, value fp64 (T,): f' inside R_q and the exact score outside, above int64 (T,): rows ranking before each
        flagged target, 0 when unflagged), CUDA tensors.  Every row of R_q ranks before every row outside it, so a
        target outside R_q keeps its exact rank count (ops.Index.rank_counts)."""
        off, rows, flags = self._targets(qdescs.shape[0], t_off, t_rows, t_flags)
        T = rows.shape[0]
        inside = torch.zeros(T, dtype=torch.uint8, device="cuda")
        value = torch.zeros(T, dtype=torch.float64, device="cuda")
        above = torch.zeros(T, dtype=torch.int64, device="cuda")
        for q0, _, _, loc, fb, _, _ in self._trunc_blocks(qdescs, m, kq, alpha, iters, tol, q_block):
            b, mm = fb.shape
            lo, hi = int(off[q0]), int(off[q0 + b])
            if hi == lo:
                continue
            o_d = torch.from_numpy(np.ascontiguousarray(off[q0:q0 + b + 1] - lo, dtype=np.int32)).to(fb.device)
            r_d = torch.from_numpy(rows[lo:hi]).to(fb.device)
            f_d = torch.from_numpy(flags[lo:hi]).to(fb.device)
            lib.call("dirb200_diffusion_trunc_rank_count", ops._ptr(loc.rows), ops._ptr(fb), b, mm, ops._ptr(o_d),
                     ops._ptr(r_d), ops._ptr(f_d), hi - lo, ops._ptr(inside[lo:hi]), ops._ptr(value[lo:hi]),
                     ops._ptr(above[lo:hi]), ops._stream())
        out = inside == 0
        if T and bool(out.any()):
            sc, ab = self.index.rank_counts(rows64(qdescs), off, rows, flags)
            value = torch.where(out, sc, value)
            above = torch.where(out & torch.from_numpy(flags != 0).to(above.device), ab, above)
        return inside.bool(), value, above
