"""NumPy model of IVF-PQ (DESIGN.md section 4.11, rules P1-P8), the oracle of deep-image-retrieval_b200/ivfpq.py and
csrc/pq.cu.  The lists (rule P1) come from ivf_model; exact scores from kmeans_model.exact_scores.

`bug` plants one of the mistakes the host tests must catch: 'fma' (fused multiply-add in the distances), 'tie_larger'
(codeword ties to the larger index), 'table_order' (table sums over t descending), 'no_list_term' (ADC without
b(q, c)), 'cand_tie_position' (candidate ties by list position instead of row), 'refine_adc' (the result ordered by
the ADC score instead of the exact one)."""
import numpy as np

import ivf_model

MS = (8, 16, 32, 64, 128)


def residuals(X, C, labels):
    """P2: fl32(x_r - c_label(r)), elementwise."""
    return (np.asarray(X, np.float32) - np.asarray(C, np.float32)[labels]).astype(np.float32)


def sample(n, train_size, seed):
    """P3: the sorted training rows and the training-set positions of the 256 initial codewords."""
    rng = np.random.default_rng(seed)
    rows = np.sort(rng.choice(n, train_size, replace=False))
    return rows, rng.choice(train_size, 256, replace=False)


def distances(S, CB, bug=None):
    """P4: dist[i, j] = sum over t ascending of fl64(S[i, t] - CB[j, t])^2, products and sums rounded separately."""
    S = np.asarray(S, np.float32).astype(np.float64)
    CB = np.asarray(CB, np.float32).astype(np.float64)
    s = np.zeros((S.shape[0], CB.shape[0]))
    for t in range(S.shape[1]):
        u = S[:, t, None] - CB[None, :, t]
        if bug == "fma":
            s = (s.astype(np.longdouble) + u.astype(np.longdouble) * u.astype(np.longdouble)).astype(np.float64)
        else:
            s = s + u * u
    return s


def nearest(S, CB, bug=None):
    """P4: the nearest codeword, ties to the smaller index."""
    dist = distances(S, CB, bug)
    if bug == "tie_larger":
        return (CB.shape[0] - 1 - np.argmin(dist[:, ::-1], axis=1)).astype(np.uint8)
    return np.argmin(dist, axis=1).astype(np.uint8)


def encode(Rs, CBs, bug=None):
    """P4 for every sub-space: Rs (n, D) residuals, CBs (M, 256, d) -> codes (n, M) uint8."""
    M, _, d = CBs.shape
    return np.stack([nearest(Rs[:, m * d:(m + 1) * d], CBs[m], bug) for m in range(M)], axis=1)


def update(Rs, codes, CBs):
    """P3: codeword j of sub-space m = fl32(s / n), s the sequential fp64 sum of its members' residuals in row order;
    no members keeps the codeword.  -> (codebooks, empty codewords)."""
    CBs = np.array(CBs, np.float32)
    M, _, d = CBs.shape
    empty = 0
    for m in range(M):
        sub = Rs[:, m * d:(m + 1) * d].astype(np.float64)
        for j in range(256):
            mem = np.nonzero(codes[:, m] == j)[0]
            if len(mem) == 0:
                empty += 1
                continue
            s = np.zeros(d)
            for r in mem:
                s = s + sub[r]
            CBs[m, j] = (s / len(mem)).astype(np.float32)
    return CBs, empty


def train(X, C, labels, M, train_size, pq_iter, seed, bug=None):
    """P3: the codebooks (M, 256, d) after pq_iter Lloyd iterations from 256 training residuals."""
    n, D = X.shape
    d = D // M
    rows, init = sample(n, train_size, seed)
    Rs = residuals(X[rows], C, labels[rows])
    CBs = Rs[init].reshape(256, M, d).transpose(1, 0, 2).copy()
    empty = 0
    for _ in range(pq_iter):
        CBs, empty = update(Rs, encode(Rs, CBs, bug), CBs)
    return CBs, empty


def tables(Qv, CBs, bug=None):
    """P5: T[q, m, j] = fl32(sum over t ascending of q_{m,t} C_m[j][t]) in fp64 (separate roundings)."""
    Qv = np.asarray(Qv, np.float32).astype(np.float64)
    M, _, d = CBs.shape
    out = np.empty((Qv.shape[0], M, 256), np.float32)
    ts = range(d - 1, -1, -1) if bug == "table_order" else range(d)
    for m in range(M):
        cb = CBs[m].astype(np.float64)
        acc = np.zeros((Qv.shape[0], 256))
        for t in ts:
            acc = acc + Qv[:, m * d + t, None] * cb[None, :, t]
        out[:, m] = acc.astype(np.float32)
    return out


def adc(Tq, b, codes, bug=None):
    """P5: s = fl32(b), then s = fl32(s + T[m][code_m]) for m ascending; codes (n, M) -> fp32 (n,)."""
    s = np.full(codes.shape[0], 0.0 if bug == "no_list_term" else b, np.float32)
    for m in range(codes.shape[1]):
        s = (s + Tq[m][codes[:, m]]).astype(np.float32)
    return s


def union_adc(Tq, probes_q, Ec_q, codes_list, perm, off, bug=None):
    """The probed rows R(q) in probe order and their ADC scores (codes_list in list order)."""
    rows, a, pos = [], [], []
    for c in probes_q:
        seg = slice(off[c], off[c + 1])
        rows.append(perm[seg])
        pos.append(np.arange(off[c], off[c + 1]))
        a.append(adc(Tq, np.float32(Ec_q[c]), codes_list[seg], bug))
    cat = lambda v, t: np.concatenate(v + [np.empty(0, t)])
    return cat(rows, np.int64), cat(a, np.float32), cat(pos, np.int64)


def candidates(rows, a, R, bug=None, pos=None):
    """P6: the first min(R, |R(q)|) rows in (a desc, row asc) order."""
    key = pos if bug == "cand_tie_position" else rows
    return rows[np.lexsort((key, -a.astype(np.float64)))[:R]]


def search(E, T, Ec, probes, codes_list, perm, off, k, R, bug=None):
    """P7 for every query -> (scores (Q, k), rows (Q, k), C_q list)."""
    Q = E.shape[0]
    sc = np.full((Q, k), -np.inf)
    ix = np.full((Q, k), -1, np.int64)
    cands = []
    for q in range(Q):
        rows, a, pos = union_adc(T[q], probes[q], Ec[q], codes_list, perm, off, bug)
        cq = candidates(rows, a, R, bug, pos)
        cands.append(cq)
        if bug == "refine_adc":
            amap = dict(zip(rows.tolist(), a.tolist()))
            o = np.lexsort((cq, -np.array([amap[r] for r in cq])))[:k]
        else:
            o = ivf_model.order(cq, E[q, cq])[:k]
        sc[q, :len(o)] = E[q, cq[o]]
        ix[q, :len(o)] = cq[o]
    return sc, ix, cands


def ranks(E, cands, t_q, t_rows):
    """P8: rank of target t of query t_q in L_q = C_q in exact order, then every other row in exact order."""
    N = E.shape[1]
    allrows = np.arange(N)
    out = np.empty(len(t_rows), np.int64)
    for i, (q, t) in enumerate(zip(t_q, t_rows)):
        before = (E[q] > E[q, t]) | ((E[q] == E[q, t]) & (allrows < t))
        a_all = int(before.sum())
        cq = cands[q]
        a_in = int(before[cq].sum())
        out[i] = a_in if np.isin(t, cq) else len(cq) + a_all - a_in
    return out

