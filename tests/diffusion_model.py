"""numpy / scipy restatement of the diffusion rules of DESIGN.md section 4.7 (the oracle of the diffusion kernels).

Every function follows one rule in fp64; `bug=` plants one plausible implementation mistake, so the tests can show
that each leaves a check."""
import numpy as np
import scipy.sparse as sp

U = 2.0 ** -53                     # unit roundoff of fp64


def gamma_n(n):
    return n * U / (1 - n * U)


def exact_scores(X, Q=None):
    """fp64 dot products of fp32 rows (each product is exact); X X^T made exactly symmetric, as exact_dot_warp is."""
    X = np.asarray(X, np.float32).astype(np.float64)
    if Q is not None:
        return np.asarray(Q, np.float32).astype(np.float64) @ X.T
    S = X @ X.T
    return np.triu(S) + np.triu(S, 1).T


def topk_lists(S, width):
    """Rule 1's lists: per row the first `width` columns by (score desc, index asc); -1 / -inf past the end."""
    n_q, n = S.shape
    idx = np.full((n_q, width), -1, np.int64)
    sc = np.full((n_q, width), -np.inf)
    cols = np.arange(n)
    for i in range(n_q):
        order = np.lexsort((cols, -S[i]))[:width]
        idx[i, :len(order)] = order
        sc[i, :len(order)] = S[i, order]
    return idx, sc


def neighbours(idx, sc, k, gamma, bug=None):
    """nn(i) (the first k entries other than i, dropped by index) with w_ij = max(s_ij, 0)^gamma -> list of dicts."""
    out = []
    for i in range(idx.shape[0]):
        d = {}
        for pos, (j, s) in enumerate(zip(idx[i], sc[i])):
            if j < 0:
                continue
            if (pos == 0) if bug == "self_by_position" else (j == i):
                continue
            if len(d) == k:
                break
            w = np.float32(max(s, 0.0)) ** np.float32(gamma) if bug == "pow32" else max(s, 0.0) ** gamma
            d[int(j)] = float(w)
        out.append(d)
    return out


def graph(idx, sc, k, gamma, bug=None):
    """Rules 2-3 -> (row_ptr int64, col int32, val fp64) with columns ascending within a row."""
    nb = neighbours(idx, sc, k, gamma, bug)
    n = len(nb)
    rows = []
    for i in range(n):
        if bug == "union":
            js = sorted(set(nb[i]) | {j for j in range(n) if i in nb[j]})
            rows.append([(j, nb[i][j] if j in nb[i] else nb[j][i]) for j in js])
        else:
            rows.append([(j, nb[i][j]) for j in sorted(nb[i]) if i in nb[j]])
    d = np.zeros(n)
    for i in range(n):
        acc = 0.0
        for _, a in rows[i]:              # ascending j
            acc += a
        d[i] = acc
    u = np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 0.0)
    row_ptr = np.zeros(n + 1, np.int64)
    col, val = [], []
    for i in range(n):
        for j, a in rows[i]:
            col.append(j)
            if bug == "dinv":
                val.append(a / d[i])
            elif bug == "asym_order":
                val.append((a * u[i]) * u[j])
            else:
                val.append(a * (u[i] * u[j]))
        row_ptr[i + 1] = len(col)
    return row_ptr, np.array(col, np.int32), np.array(val, np.float64)


def to_csr(row_ptr, col, val, n):
    return sp.csr_matrix((np.asarray(val, np.float64), np.asarray(col, np.int64), np.asarray(row_ptr, np.int64)), shape=(n, n))


def seeds(idx, sc, n, gamma):
    """Rule 4: y [N][Q]."""
    y = np.zeros((n, idx.shape[0]))
    for q in range(idx.shape[0]):
        for j, s in zip(idx[q], sc[q]):
            if j >= 0:
                y[j, q] = max(s, 0.0) ** gamma
    return y


def cg(S, y, alpha, iters, tol, bug=None):
    """Rule 5 for one query: -> (f, iterations, final recurrence ||r||)."""
    def op(p):
        sp_ = S @ p
        if bug == "drop_row":
            sp_[S.shape[0] // 2] = 0.0
        return p - alpha * sp_

    def done(rr, yy):
        return rr <= tol if bug == "rr_tol" else np.sqrt(rr) <= tol * np.sqrt(yy)

    f = np.zeros_like(y)
    r, p = y.copy(), y.copy()
    rr = yy = float(r @ r)
    if yy == 0 or done(rr, yy):
        return f, 0, np.sqrt(rr)
    for it in range(1, iters + 1):
        ap = op(p)
        al = rr / float(p @ ap)
        f = f + al * p
        r = r - al * ap
        rn = float(r @ r)
        beta, rr = rn / rr, rn
        if done(rr, yy):
            return f, it, np.sqrt(rr)
        p = r + beta * p
    return f, iters, np.sqrt(rr)


def solve(S, Y, alpha, iters, tol, bug=None):
    """All columns of Y -> (f [Q][N], iterations (Q,), residuals (Q,))."""
    out = [cg(S, Y[:, q], alpha, iters, tol, bug) for q in range(Y.shape[1])]
    return np.stack([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out])


def true_residual(S, y, f, alpha):
    return float(np.linalg.norm(y - (f - alpha * (S @ f))))


def dense_solve(S, y, alpha):
    return np.linalg.solve(np.eye(S.shape[0]) - alpha * S.toarray(), y)


def ranking(f):
    """Rule 6: f descending, ties -> lower index, -0 == +0."""
    return np.argsort(-f, kind="stable")


def rank_counts(f, rows, flags):
    """Rows ranking before each flagged target under rule 6 (0 for unflagged targets)."""
    idx = np.arange(f.shape[0])
    return np.array([int(((f > f[t]) | ((f == f[t]) & (idx < t))).sum()) if fl else 0 for t, fl in zip(rows, flags)],
                    np.int64)


def diffuse(X, Q, k, kq, gamma, alpha, iters, tol, bug=None):
    """The whole chain on host rows -> (f [Q][N], iterations, residuals, (row_ptr, col, val))."""
    n = X.shape[0]
    idx, sc = topk_lists(exact_scores(X), k + 1)
    g = graph(idx, sc, k, gamma, bug)
    qi, qs = topk_lists(exact_scores(X, Q), kq)
    f, it, res = solve(to_csr(*g, n), seeds(qi, qs, n, gamma), alpha, iters, tol, bug)
    return f, it, res, g


def planted_manifold(seed=0, chains=6, length=24, step_deg=9.0, distractors=150, dim=64, noise=0.01):
    """Chains of points along great circles (consecutive points step_deg apart) among random distractors.  The query
    of chain c sits at its start; every point of the chain is a positive, but its far end (more than 90 degrees from
    the query) scores below the distractors: reachable only through the chain.  -> (X, Q, positives per query)."""
    r = np.random.RandomState(seed)
    pts, pos, queries = [], [], []
    for c in range(chains):
        basis, _ = np.linalg.qr(r.standard_normal((dim, 2)))
        u, v = basis[:, 0], basis[:, 1]
        first = len(pts)
        for t in range(length):
            a = np.deg2rad(step_deg * (t + 1))
            pts.append(np.cos(a) * u + np.sin(a) * v + noise * r.standard_normal(dim))
        pos.append(list(range(first, first + length)))
        queries.append(u + noise * r.standard_normal(dim))
    pts += list(r.standard_normal((distractors, dim)))
    X = np.array(pts)
    perm = r.permutation(X.shape[0])
    inv = np.argsort(perm)
    X = X[perm]
    pos = [sorted(int(inv[p]) for p in ps) for ps in pos]
    nrm = lambda a: (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)
    return nrm(X), nrm(np.array(queries)), pos


def average_precision(order, positives):
    """AP of the ranking `order` (row indices, best first) with the repository's trapezoid formula."""
    from dirb200.datasets import compute_average_precision
    rank = np.empty(order.shape[0], np.int64)
    rank[order] = np.arange(order.shape[0])
    return float(compute_average_precision(np.sort(rank[np.asarray(positives)])))
