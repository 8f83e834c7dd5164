"""NumPy model of the graph search (DESIGN.md section 4.12, rules G2-G8).

Scores are exact_dot_warp's (kmeans_model.exact_scores, rule G1); the kNN lists of rule G2 come from the exact search.
`bug` plants one of the mistakes the host tests must catch: 'detour_le' (p <= j in G3), 'rev_reversed' (Rev ordered by
source descending), 'parents_ignore_flag' (parents taken from B whether expanded or not), 'row_desc' (ties to the
larger row), 'dedupe_against_b' (N_t filtered against B instead of V)."""
import numpy as np


def knn_lists(idx, K):
    """Rule G2: each row's list of K + 1 entries without the row itself, or without its last entry when the row is
    not in it -> int64 (N, K)."""
    idx = np.asarray(idx, np.int64)[:, :K + 1]
    out = np.empty((idx.shape[0], K), np.int64)
    for r in range(idx.shape[0]):
        L = idx[r].tolist()
        if r in L:
            L.remove(r)
        else:
            L = L[:K]
        out[r] = L
    return out


def detours(knn, bug=None):
    """Rule G3: det[r, j] = |{i < j : n_j is in knn(n_i) at a position p < j}| (0 where n_j = -1)."""
    n, K = knn.shape
    out = np.zeros((n, K), np.int64)
    if K == 0:
        return out
    pos = np.arange(K)
    pj = (pos[:, None] <= pos[None, :]) if bug == "detour_le" else (pos[:, None] < pos[None, :])    # [p, j]
    ij = pos[:, None] < pos[None, :]                                                                # [i, j]
    step = max(1, (1 << 22) // (K ** 3))
    for r0 in range(0, n, step):
        L = knn[r0:r0 + step]
        NL = np.where(L[..., None] >= 0, knn[np.maximum(L, 0)], -1)                 # [c, i, p]
        hit = ((NL[:, :, :, None] == L[:, None, None, :]) & pj[None, None]).any(2)   # [c, i, j]
        hit &= ij[None] & (L[:, :, None] >= 0) & (L[:, None, :] >= 0)
        out[r0:r0 + step] = hit.sum(1)
    return out


def forward(knn, degree, bug=None):
    """Rule G4: F(r) = the `degree` valid entries of knn(r) with the fewest detours, (detours asc, position asc),
    -1 padded -> int64 (N, degree)."""
    n, K = knn.shape
    det = detours(knn, bug)
    key = np.where(knn >= 0, det * 256 + np.arange(K), np.iinfo(np.int64).max)
    order = np.argsort(key, axis=1, kind="stable")
    F = np.full((n, degree), -1, np.int64)
    m = min(degree, K)
    srt = np.take_along_axis(knn, order, 1)[:, :m]
    ok = np.take_along_axis(key, order, 1)[:, :m] != np.iinfo(np.int64).max
    F[:, :m] = np.where(ok, srt, -1)
    return F


def reverse(F, bug=None):
    """Rule G5: Rev(r) = the s with r in F(s), ordered by (r's position in F(s) asc, s asc) -> list of lists."""
    n, degree = F.shape
    s, p = np.nonzero(F >= 0)
    t = F[s, p]
    order = np.lexsort((-s if bug == "rev_reversed" else s, p, t))
    rev = [[] for _ in range(n)]
    for e in order:
        rev[t[e]].append(int(s[e]))
    return rev


def merge(F, rev, degree):
    """Rule G5: G(r) = F(r)[0 : degree/2], then Rev(r) entries not yet present, then the rest of F(r) without
    repeats, up to `degree` entries, -1 padded -> int64 (N, degree)."""
    n = F.shape[0]
    G = np.full((n, degree), -1, np.int64)
    h = degree // 2
    for r in range(n):
        f = [int(c) for c in F[r] if c >= 0]
        g = f[:h]
        seen = set(g)
        for c in rev[r] + f[h:]:
            if len(g) == degree:
                break
            if c not in seen:
                g.append(c)
                seen.add(c)
        G[r, :len(g)] = g
    return G


def build(knn_idx, K, degree, bug=None):
    """Rules G2-G5 from the exact top-(K + 1) lists (or a caller's lists in that format)."""
    F = forward(knn_lists(knn_idx, K), degree, bug)
    return merge(F, reverse(F, bug), degree)


def entry(n, n_entry, seed):
    """Rule G6's sample."""
    return np.sort(np.random.default_rng(seed).choice(n, min(n, n_entry), replace=False))


def _order(e, rows, bug=None):
    return sorted(rows, key=(lambda r: (-e[r], -r)) if bug == "row_desc" else (lambda r: (-e[r], r)))


def seeds(e, E, n_seeds):
    """Rule G6: the best n_seeds rows of the sample E for the query with scores e (over all rows)."""
    return _order(e, [int(r) for r in E])[:n_seeds]


def traverse(e, G, sd, itopk, width, max_iter, bug=None):
    """Rule G7 for one query (e: its exact scores over all rows) -> (V in arrival order, B, iterations)."""
    V = list(sd)
    inV = set(V)
    expanded = set()
    B = _order(e, V, bug)[:itopk]
    it = 0
    while it < max_iter:
        par = B[:width] if bug == "parents_ignore_flag" else [r for r in B if r not in expanded][:width]
        if not par:
            break
        expanded.update(par)
        it += 1
        new = []
        for p in par:
            for c in G[p]:
                c = int(c)
                if c < 0 or c in new or (c in B if bug == "dedupe_against_b" else c in inV):
                    continue
                new.append(c)
        inV.update(new)
        V += new
        B = _order(e, B + new, bug)[:itopk]
    return V, B, it


def search(e, G, sd, k, itopk, width, max_iter, bug=None):
    """Rule G7's result for one query -> (scores (k,), rows (k,), V, iterations), padded (-inf, -1)."""
    V, B, it = traverse(e, G, sd, itopk, width, max_iter, bug)
    sc = np.full(k, -np.inf)
    ix = np.full(k, -1, np.int64)
    top = B[:k]
    sc[:len(top)] = e[top]
    ix[:len(top)] = top
    return sc, ix, V, it


def ranks(e, V, targets):
    """Rule G8 for one query: the rank of each target in V in exact order, then every other row in exact order."""
    n = e.shape[0]
    rows = np.arange(n)
    inV = np.zeros(n, bool)
    inV[np.asarray(V, np.int64)] = True
    out = []
    for t in targets:
        before = (e > e[t]) | ((e == e[t]) & (rows < t))
        a_all, a_in = int(before.sum()), int(before[inV].sum())
        out.append(a_in if inV[t] else len(V) + a_all - a_in)
    return np.asarray(out, np.int64)
