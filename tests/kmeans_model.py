"""numpy restatement of spherical k-means, rules K1-K7 of DESIGN.md section 4.9 (the oracle of
deep-image-retrieval_b200/cluster.py and csrc/kmeans.cu).

Every function follows one rule; `bug=` plants one plausible implementation mistake, so the tests can show that each
leaves a check."""
import numpy as np

CHUNK = 256          # K5: rows per chunk of a centre sum
NORM_THREADS = 256   # K5: partial sums of ||s||^2
FIX = 2.0 ** 32      # K6 / K7: fixed-point units of 2^-32


def exact_scores(A, B):
    """K1: exact_dot_warp of csrc/exact_dot.cuh for every pair (a, b): float4 column group g goes to lane g % 32, each
    lane adds its fp64 products in column order, then an xor-shuffle tree (offsets 16, 8, 4, 2, 1) adds the lanes."""
    A = np.ascontiguousarray(A, np.float32)
    B = np.ascontiguousarray(B, np.float32)
    n, d = A.shape
    k = B.shape[0]
    groups = d // 4
    steps = -(-groups // 32)
    pad = steps * 128 - d
    Ap = np.pad(A, ((0, 0), (0, pad))).astype(np.float64).reshape(n, steps, 32, 4)
    Bp = np.pad(B, ((0, 0), (0, pad))).astype(np.float64).reshape(k, steps, 32, 4)
    valid = (np.arange(steps)[:, None] * 32 + np.arange(32)[None, :]) < groups
    out = np.empty((n, k))
    rows = max(1, (1 << 22) // max(k * 32, 1))
    lanes = np.arange(32)
    for r0 in range(0, n, rows):
        a = Ap[r0:r0 + rows]
        acc = np.zeros((a.shape[0], k, 32))
        for t in range(steps):
            for c in range(4):
                p = a[:, None, t, :, c] * Bp[None, :, t, :, c]
                acc = acc + p if valid[t].all() else np.where(valid[t], acc + p, acc)
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[..., lanes ^ o]
        out[r0:r0 + rows] = acc[..., 0]
    return out


def assign(E, bug=None):
    """K2: label(i) = the smallest c maximising E[i, c] (bug 'ties_last': the largest), score(i) = that E."""
    if bug == "ties_last":
        lab = E.shape[1] - 1 - np.argmax(E[:, ::-1], axis=1)
    else:
        lab = np.argmax(E, axis=1)
    return lab.astype(np.int64), E[np.arange(E.shape[0]), lab]


def band_threshold(M, eps16, bug=None):
    """K3: t = M - 2 eps16 in fp64, rounded DOWN to fp32 (bug 'band1': M - eps16; bug 'round_nearest': rounded to
    nearest)."""
    x = float(M) - (1.0 if bug == "band1" else 2.0) * float(eps16)
    f = np.float32(x)
    if bug != "round_nearest" and float(f) > x:
        f = np.nextafter(f, np.float32(-np.inf))
    return f


def candidates(F_row, eps16, cap, bug=None):
    """K3 for one row: F_row the fp32 fp16-path scores of the K centres.  G[g] = max over the centres 32g .. 32g+31,
    M = max G, the groups with G >= t; more than cap groups -> every centre.  -> (centres, n_groups, full)."""
    K = F_row.shape[0]
    ng = -(-K // 32)
    G = np.full(ng * 32, -np.inf, np.float32)
    G[:K] = F_row
    G = G.reshape(ng, 32).max(axis=1)
    t = band_threshold(G.max(), eps16, bug)
    groups = np.nonzero(G >= t)[0]
    if len(groups) > cap:
        return np.arange(K), len(groups), True
    c = (groups[:, None] * 32 + np.arange(32)[None, :]).ravel()
    return c[c < K], len(groups), False


def nearest(E, F, eps16, cap=16, bug=None):
    """K2 through K3: the best exact score among each row's candidates, ties to the smallest centre."""
    lab = np.empty(E.shape[0], np.int64)
    for i in range(E.shape[0]):
        c, _, _ = candidates(F[i], eps16, cap, bug)
        e = E[i, c]
        lab[i] = c[np.nonzero(e == e.max())[0][0]]
    return lab, E[np.arange(E.shape[0]), lab]


def relocate(labels, scores, k, bug=None):
    """K4: each empty cluster, ascending, takes the row of lowest (score, row) among the rows whose cluster still has
    >= 2 rows, the sizes updated after each move (bug 'singleton': a row of a 1-row cluster qualifies).
    -> (labels, moves)."""
    labels = labels.copy()
    counts = np.bincount(labels, minlength=k)
    order = np.lexsort((np.arange(len(labels)), scores))
    moves = 0
    least = 1 if bug == "singleton" else 2
    for c in np.nonzero(counts == 0)[0]:
        for r in order:
            l = labels[r]
            if counts[l] >= least:
                counts[l] -= 1
                labels[r] = c
                counts[c] += 1
                moves += 1
                break
    return labels, moves


def centre_sum(X, members, bug=None):
    """K5: s = the fp64 sum of the members' rows (ascending) in chunks of CHUNK rows, each chunk summed sequentially,
    the chunk sums added in chunk order (bug 'order': one sequential sum in descending row order)."""
    X = np.asarray(X, np.float32)
    s = np.zeros(X.shape[1])
    if bug == "order":
        for r in members[::-1]:
            s = s + X[r].astype(np.float64)
        return s
    for c0 in range(0, len(members), CHUNK):
        acc = np.zeros(X.shape[1])
        for r in members[c0:c0 + CHUNK]:
            acc = acc + X[r].astype(np.float64)
        s = s + acc
    return s


def norm2(s):
    """K5: ||s||^2 - partial p_t = sum over the columns t, t + 256, ... in order of s_j * s_j (each product rounded),
    then p_t += p_{t + h} for h = 128, 64, ..., 1; the result is p_0."""
    p = np.zeros(NORM_THREADS)
    for j0 in range(0, len(s), NORM_THREADS):
        seg = s[j0:j0 + NORM_THREADS]
        p[:len(seg)] = p[:len(seg)] + seg * seg
    h = NORM_THREADS // 2
    while h:
        p[:h] = p[:h] + p[h:2 * h]
        h //= 2
    return p[0]


def update(X, labels, C, bug=None):
    """K5: each centre becomes fl32(s / sqrt(||s||^2)); s = 0 keeps the old centre. -> (centres, zero sums)."""
    C = np.array(C, np.float32)
    zero = 0
    for c in range(C.shape[0]):
        s = centre_sum(X, np.nonzero(labels == c)[0], bug)
        ss = norm2(s)
        if ss == 0.0:
            zero += 1
            continue
        C[c] = (s / np.sqrt(ss)).astype(np.float32)
    return C, zero


def objective_units(scores):
    """K6: the sum of rint(score * 2^32), an exact integer."""
    return int(np.rint(np.asarray(scores) * FIX).astype(np.int64).sum())


def kmeans_pp(X, k, seed, bug=None):
    """K7: D^2 sampling with every draw taken up front from RandomState(seed): the first row randint(N), then
    K - 1 values u of random_sample().  Weights w_i = rint(max(0, 2 - 2 e(x_i, nearest chosen row)) * 2^32), chosen
    rows 0 (bug 'not_zeroed': they keep their weight); T = sum w, t = min(floor(u * float(T)), T - 1); the next row is
    the first whose inclusive prefix exceeds t.  T = 0 -> ValueError."""
    X = np.asarray(X, np.float32)
    n = X.shape[0]
    rs = np.random.RandomState(seed)
    first = int(rs.randint(n))
    u = rs.random_sample(k - 1)
    chosen = [first]
    flag = np.zeros(n, bool)
    flag[first] = True
    best = None
    for j in range(1, k):
        e = exact_scores(X, X[chosen[-1]][None])[:, 0]
        best = e if best is None else np.maximum(best, e)
        w = np.rint(np.maximum(0.0, 2.0 - 2.0 * best) * FIX).astype(np.int64)
        if bug != "not_zeroed":
            w[flag] = 0
        T = int(w.sum())
        if T == 0:
            raise ValueError("fewer than k distinct rows")
        t = min(int(np.floor(u[j - 1] * float(T))), T - 1)
        r = int(np.searchsorted(np.cumsum(w), t, side="right"))
        chosen.append(r)
        flag[r] = True
    return np.array(chosen, np.int64)


def initial_centres(X, k, init, seed, bug=None):
    X = np.asarray(X, np.float32)
    if isinstance(init, str):
        rows = kmeans_pp(X, k, seed, bug) if init == "k-means++" else np.random.RandomState(seed).permutation(len(X))[:k]
        return X[rows].copy()
    return np.array(init, np.float32)


def fit(X, k, init="k-means++", max_iter=20, seed=0, bug=None, scores=exact_scores):
    """K6: assign, then (unless the assignment repeats the previous one, or max_iter iterations ran) relocate and
    update; the returned labels / scores always belong to the returned centres."""
    X = np.asarray(X, np.float32)
    C = initial_centres(X, k, init, seed, bug)
    prev, n_iter, relocations, zero_sums = None, 0, 0, 0
    while True:
        labels, sc = assign(scores(X, C), bug)
        if (prev is not None and np.array_equal(labels, prev)) or n_iter == max_iter:
            break
        if (np.bincount(labels, minlength=k) == 0).any():
            labels, m = relocate(labels, sc, k, bug)
            relocations += m
        C, z = update(X, labels, C, bug)
        zero_sums += z
        prev = labels
        n_iter += 1
    return dict(centres=C, labels=labels, scores=sc, n_iter=n_iter, objective=objective_units(sc) / FIX,
                relocations=relocations, zero_sums=zero_sums)
