"""NumPy model of the inverted-file search (DESIGN.md section 4.10, rules I1-I7) and of its device-built tile table.

E = exact scores (kmeans_model.exact_scores restates exact_dot_warp, rule I1).  `bug` plants one of the mistakes the
host tests must catch: 'drop_last_tile', 'cell_off_shift', 'tie_by_position', 'probe_tie_larger', 'no_band',
'a_in_all_rows'."""
import numpy as np

TILE = 128


def build(labels, K, bug=None):
    """Rule I2: perm (list position -> row, list ascending then row ascending) and cell_off (K + 1)."""
    labels = np.asarray(labels, np.int64)
    perm = np.argsort(labels, kind="stable")
    off = np.zeros(K + 1, np.int64)
    np.cumsum(np.bincount(labels, minlength=K), out=off[1:])
    if bug == "cell_off_shift":
        off[1:-1] += 1
    return perm, off


def probe(Ec, nprobe, bug=None):
    """Rule I3: the nprobe best centres per query, score desc, ties to the smaller centre."""
    K = Ec.shape[1]
    if not 1 <= nprobe <= K:
        raise ValueError("nprobe must be in [1, %d]" % K)
    c = np.arange(K)
    out = np.empty((Ec.shape[0], nprobe), np.int64)
    for q in range(Ec.shape[0]):
        tie = -c if bug == "probe_tie_larger" else c
        out[q] = np.lexsort((tie, -Ec[q]))[:nprobe]
    return out


def union(probes_q, perm, off):
    """R(q): the rows of the probed lists."""
    return np.concatenate([perm[off[c]:off[c + 1]] for c in probes_q] + [np.empty(0, np.int64)])


def order(rows, scores, bug=None, pos=None):
    """(e desc, row asc); the planted bug orders ties by list position instead of row."""
    key = pos if bug == "tie_by_position" else rows
    return np.lexsort((key, -scores))


def search(E, probes, perm, off, k, bug=None):
    """Rule I4: the first k rows of R(q) in (e desc, row asc) order, padded with (-inf, -1)."""
    Q = E.shape[0]
    sc = np.full((Q, k), -np.inf)
    ix = np.full((Q, k), -1, np.int64)
    inv = np.empty_like(perm)
    inv[perm] = np.arange(perm.shape[0])
    for q in range(Q):
        R = union(probes[q], perm, off)
        o = order(R, E[q, R], bug, inv[R])[:k]
        sc[q, :o.shape[0]] = E[q, R[o]]
        ix[q, :o.shape[0]] = R[o]
    return sc, ix


def candidates(F, probes, perm, off, k, band, bug=None):
    """Rule I5 with the baseline seed: thr_q = k-th largest group maximum (groups of 32 list rows, per probed list) of
    the fp16-path scores F, -inf with fewer than k groups; the candidates are the probed rows with F >= thr_q - band."""
    out = []
    for q in range(F.shape[0]):
        gm = []
        for c in probes[q]:
            seg = F[q, perm[off[c]:off[c + 1]]]
            gm += [seg[i:i + 32].max() for i in range(0, seg.shape[0], 32)]
        gm = np.sort(np.asarray(gm, np.float32))[::-1]
        t = gm[k - 1] if gm.shape[0] >= k else np.float32(-np.inf)
        thr = np.float32(t - (np.float32(0) if bug == "no_band" else np.float32(band)))
        R = union(probes[q], perm, off)
        out.append(R[F[q, R] >= thr])
    return out


def tile_table(probes, off, bug=None):
    """Mirror of ivf_mark / _list_count / _scan / _list_fill (csrc/search.cu): slots (segment row -> query, -1 = padding)
    and tiles (A row, B row, column tile, valid rows, valid columns), lists in order, queries ascending, m fastest."""
    K = off.shape[0] - 1
    Q = probes.shape[0]
    members = [[] for _ in range(K)]
    for q in range(Q):
        for c in probes[q]:
            members[c].append(q)
    slots, tiles = [], []
    for c in range(K):
        n = int(off[c + 1] - off[c])
        pc = len(members[c])
        if n == 0 or pc == 0:
            continue
        s0 = len(slots)
        padded = -(-pc // TILE) * TILE
        slots += members[c] + [-1] * (padded - pc)
        nt = -(-n // TILE)
        if bug == "drop_last_tile" and n % TILE:
            nt -= 1
        mt = padded // TILE
        for t in range(mt * nt):
            m, nn = t % mt, t // mt
            tiles.append((s0 + TILE * m, int(off[c]) + TILE * nn, nn, min(TILE, pc - TILE * m), min(TILE, n - TILE * nn)))
    return np.asarray(slots, np.int64), tiles


def covered_pairs(slots, tiles, perm):
    """Every (query, row) a tile table issues, with the masks of the epilogues applied."""
    out = []
    for a, b, _, mv, nv in tiles:
        for r in range(mv):
            for j in range(nv):
                out.append((int(slots[a + r]), int(perm[b + j])))
    return out


def ranks(E, probes, perm, off, t_q, t_rows, bug=None):
    """Rule I7: rank of target t of query t_q[t] in L_q = R(q) in exact order, then every other row in exact order."""
    N = E.shape[1]
    rows = np.arange(N)
    out = np.empty(t_rows.shape[0], np.int64)
    for i, (q, t) in enumerate(zip(t_q, t_rows)):
        R = union(probes[q], perm, off)
        before = (E[q] > E[q, t]) | ((E[q] == E[q, t]) & (rows < t))
        a_all = int(before.sum())
        a_in = a_all if bug == "a_in_all_rows" else int(before[R].sum())
        out[i] = a_in if np.isin(t, R) else R.shape[0] + a_all - a_in
    return out
