"""numpy / scipy restatement of truncated diffusion, rules T1-T6 of DESIGN.md section 4.7 (the oracle of
csrc/diffusion_trunc.cu), on the graph of tests/diffusion_model.py.

Every function follows one rule in fp64 with the kernels' summation order; `bug=` plants one plausible implementation
mistake, so the tests can show that each leaves a check."""
import numpy as np
import scipy.sparse as sp

import diffusion_model as M


def weights(idx, sc, k, gamma):
    """Rules 2-3 before normalisation: (row_ptr, col, A) of the mutual-kNN graph, the CSR of M.graph."""
    nb = M.neighbours(idx, sc, k, gamma)
    row_ptr, col, val = [0], [], []
    for i in range(len(nb)):
        for j in sorted(nb[i]):
            if i in nb[j]:
                col.append(j)
                val.append(nb[i][j])
        row_ptr.append(len(col))
    return np.array(row_ptr, np.int64), np.array(col, np.int32), np.array(val, np.float64)


def region(list_idx, m, bug=None):
    """T1: R_q = the first m' list entries, local numbering by ascending global index -> (rows, list position of each)."""
    r = np.asarray(list_idx[:m], np.int64)
    order = np.arange(r.size) if bug == "list_order" else np.argsort(r, kind="stable")
    return r[order], order


def subgraph(W, rows, bug=None):
    """T2-T3 -> (row_ptr, local col, A', d', u', S') for the local rows `rows` (ascending global index)."""
    row_ptr, col, a = W
    at = {int(g): l for l, g in enumerate(rows)}
    lrp, lcol, la, d = [0], [], [], np.zeros(rows.size)
    for l, g in enumerate(rows):
        acc = 0.0
        for e in range(row_ptr[g], row_ptr[g + 1]):          # ascending global j
            j = int(col[e])
            if bug == "global_degree":
                acc += a[e]
            if j in at:
                lcol.append(at[j])
                la.append(a[e])
                if bug != "global_degree":
                    acc += a[e]
        d[l] = acc
        lrp.append(len(lcol))
    u = np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 0.0)
    lcol = np.array(lcol, np.int32)
    la = np.array(la, np.float64)
    rr = np.repeat(np.arange(rows.size), np.diff(lrp))
    if bug == "no_renorm":                                    # the global S restricted to R_q
        ug = global_u(W)
        s = la * (ug[rows[rr]] * ug[rows[lcol]])
    else:
        s = la * (u[rr] * u[lcol])
    return np.array(lrp, np.int64), lcol, la, d, u, s


def global_u(W):
    row_ptr, _, a = W
    d = np.array([sum(a[row_ptr[i]:row_ptr[i + 1]], 0.0) for i in range(row_ptr.size - 1)])
    return np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 0.0)


def seeds(list_idx, list_sc, rows, pos, kq, gamma, bug=None):
    """T4: y' = max(s, 0)^gamma at the first kq list entries (their local rows), 0 elsewhere."""
    if kq > rows.size:
        raise ValueError("kq exceeds m'")
    y = np.zeros(rows.size)
    for l, p in enumerate(pos):
        if p < kq:
            y[l] = max(list_sc[p], 0.0) ** gamma
    if bug == "outside_seeds":              # the global seed vector read at the local numbers: rows outside R_q
        yg = {int(list_idx[p]): max(list_sc[p], 0.0) ** gamma for p in range(kq)}
        y = np.array([yg.get(l, 0.0) for l in range(rows.size)])
    return y


def solve_one(W, list_idx, list_sc, m, kq, gamma, alpha, iters, tol, bug=None):
    """T1-T5 for one query -> (rows, f', iterations, residual, (row_ptr, col, A', d', u', S'), y')."""
    m = min(m, len(list_idx))
    rows, pos = region(list_idx, m, bug)
    g = subgraph(W, rows, bug)
    y = seeds(list_idx, list_sc, rows, pos, kq, gamma, bug)
    S = sp.csr_matrix((g[5], g[1].astype(np.int64), g[0]), shape=(rows.size, rows.size))
    f, it, res = M.cg(S, y, alpha, iters, tol)
    return rows, f, it, res, g, y


def ranking(rows, f, exact_list, bug=None):
    """T6: the rows of R_q by f' descending (ties -> lower global index, -0 == +0), then the rest of the exact list."""
    if bug == "outside_by_index":
        rest = np.sort(np.setdiff1d(exact_list, rows))
    else:
        inr = set(int(r) for r in rows)
        rest = np.array([j for j in exact_list if int(j) not in inr], np.int64)
    order = np.lexsort((rows, -(f + 0.0)))
    return np.concatenate([rows[order], rest]).astype(np.int64)


def diffuse(X, Q, k, kq, gamma, alpha, iters, tol, m, bug=None):
    """The whole chain on host rows -> per query (rows, f', iterations, residual, subgraph, y') and the exact lists."""
    n = X.shape[0]
    idx, sc = M.topk_lists(M.exact_scores(X), k + 1)
    W = weights(idx, sc, k, gamma)
    qi, qs = M.topk_lists(M.exact_scores(X, Q), n)
    out = [solve_one(W, qi[q], qs[q], m, kq, gamma, alpha, iters, tol, bug) for q in range(Q.shape[0])]
    return out, qi, qs


def full_ranks(rows, f, exact_list, bug=None):
    """Rank (position) of every row under T6 -> int64 (N,)."""
    order = ranking(rows, f, exact_list, bug)
    rank = np.empty(order.size, np.int64)
    rank[order] = np.arange(order.size)
    return rank
