"""numpy restatement of the range search, the triangular self-join and its groups, rules J1-J6 of DESIGN.md section 4.8
(the oracle of the join path of csrc/search.cu, the PERS_EPI_SIM_JOIN epilogue of csrc/conv_pers.cuh and csrc/join.cu).

Scores come in two matrices: E, the exact scores (rule J1), and F, the fp32 scores of the fp16 tensor-core path, with
|F - E| <= eps16.  Every function follows one rule; `bug=` plants one plausible implementation mistake, so the tests
can show that each leaves a check."""
import math

import numpy as np

TILE = 128


def threshold(tau, eps16, bug=None):
    """J5: tau - eps16 in fp64, rounded DOWN to fp32 (bug 'round_nearest': rounded to nearest)."""
    x = float(tau) - float(eps16)
    f = np.float32(x)
    if bug != "round_nearest" and float(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return f


def tri_tiles(m_tiles, n_tiles):
    """Number of tiles of a self-join launch: the tiles (m, n) with n >= m of an m_tiles x n_tiles grid."""
    return m_tiles * n_tiles - m_tiles * (m_tiles - 1) // 2


def decode_tri(t, m_tiles, bug=None):
    """decode_tile_tri of conv_pers.cuh: linear tile t -> (m, n), m fastest; column n < m_tiles holds n + 1 tiles.
    bug 'off_diagonal': the schedule starts at n >= m + 1 (the diagonal tiles are never run)."""
    if bug == "off_diagonal":                      # columns n hold min(n, m_tiles) tiles m = 0 .. n - 1
        n = 1
        while True:
            h = min(n, m_tiles)
            if t < h:
                return t, n
            t -= h
            n += 1
    mt = m_tiles
    tri = mt * (mt + 1) // 2
    if t < tri:
        n = int((math.sqrt(8.0 * t + 1.0) - 1.0) * 0.5)
        while n * (n + 1) // 2 > t:
            n -= 1
        while (n + 1) * (n + 2) // 2 <= t:
            n += 1
        return t - n * (n + 1) // 2, n
    u = t - tri
    return u % mt, mt + u // mt


def block_tiles(M, ncols, bug=None):
    """The (m, n) tiles a self-join block of M rows against ncols columns launches."""
    mt, nt = -(-M // TILE), -(-ncols // TILE)
    return [decode_tri(t, mt, bug) for t in range(tri_tiles(mt, nt))]


def _order(rows, scores):
    """(e desc, row asc)."""
    o = np.lexsort((rows, -scores))
    return rows[o], scores[o]


def range_search(E, F, tau, eps16):
    """J2 through J5: candidates F >= thr, kept e >= tau, lists by (e desc, row asc) -> CSR (off, rows, scores)."""
    thr = threshold(tau, eps16)
    off, rows, sc = [0], [], []
    for q in range(E.shape[0]):
        r = np.nonzero(F[q] >= thr)[0]
        r = r[E[q, r] >= tau]
        r, s = _order(r.astype(np.int64), E[q, r])
        rows.append(r)
        sc.append(s)
        off.append(off[-1] + len(r))
    return np.array(off, np.int64), np.concatenate(rows + [np.zeros(0, np.int64)]), np.concatenate(sc + [np.zeros(0)])


def filter_block(F, thr, r0, M, col0, cap, tri, bug=None):
    """The filter pass of one block: per row the first min(count, cap) columns (in some order) and the exact count.
    tri: the self-join epilogue over the launched tiles, col > row (bug 'keep_diagonal': col >= row)."""
    N = F.shape[1]
    lists, counts = [], []
    allowed = None
    if tri:
        allowed = np.zeros((M, N - col0), bool)
        for m, n in block_tiles(M, N - col0, bug):
            allowed[m * TILE:(m + 1) * TILE, n * TILE:(n + 1) * TILE] = True
    for q in range(M):
        c = np.nonzero(F[r0 + q, col0:] >= thr)[0]
        if tri:
            c = c[allowed[q, c]]
            c = c[c >= q] if bug == "keep_diagonal" else c[c > q]
        counts.append(len(c))
        lists.append(c[:cap] + col0)
    return lists, counts


def join_block(E, F, tau, eps16, r0, M, col0, cap, tri, bug=None):
    """J6 for one block: an overflowed list re-runs the block at the exact count (bug 'truncate': keeps the truncated
    lists without an error) -> per row (rows, scores) ordered."""
    thr = threshold(tau, eps16, bug)
    lists, counts = filter_block(F, thr, r0, M, col0, cap, tri, bug)
    if max(counts, default=0) > cap and bug != "truncate":
        lists, counts = filter_block(F, thr, r0, M, col0, max(counts), tri, bug)
    out = []
    for q in range(M):
        r = np.asarray(lists[q], np.int64)
        s = E[r0 + q, r]
        keep = s >= tau
        out.append(_order(r[keep], s[keep]))
    return out


def self_join(E, F, tau, eps16, row_block=None, cap=None, bug=None):
    """J3: pairs (i, j), i < j, e >= tau, CSR by i, blocks of row_block rows (a multiple of 128) -> (off, cols, scores)."""
    N = E.shape[0]
    step = row_block or max(N, 1)
    cap = cap or max(N, 1)
    lists = []
    for i0 in range(0, N, step):
        lists += join_block(E, F, tau, eps16, i0, min(step, N - i0), i0, cap, True, bug)
    off = np.cumsum([0] + [len(r) for r, _ in lists]).astype(np.int64)
    cols = np.concatenate([r for r, _ in lists] + [np.zeros(0, np.int64)])
    sc = np.concatenate([s for _, s in lists] + [np.zeros(0)])
    return off, cols, sc


def components(off, cols, n, bug=None):
    """J4: labels = the smallest row of each component (min-label union-find: hook the larger root to the smaller).
    bug 'first_seen': components numbered in the order they are first met."""
    parent = np.arange(n, dtype=np.int64)

    def root(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for i in range(n):
        for j in cols[off[i]:off[i + 1]]:
            a, b = root(i), root(int(j))
            if a != b:
                parent[max(a, b)] = min(a, b)
    labels = np.array([root(i) for i in range(n)], np.int64)
    if bug == "first_seen":
        seen = {}
        labels = np.array([seen.setdefault(int(l), len(seen)) for l in labels], np.int64)
    return labels


def groups(labels):
    """J4: components of >= 2 rows by ascending label, members ascending -> list of int64 arrays."""
    out = []
    for l in np.unique(labels):
        m = np.nonzero(labels == l)[0]
        if len(m) >= 2:
            out.append(m.astype(np.int64))
    return out
