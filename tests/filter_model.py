"""NumPy model of the filtered exact search (DESIGN.md section 4.13, rules F1-F6) on top of tests/search_model.py.
TEST INFRASTRUCTURE: it restates the ALGORITHM - allow bitmaps, the seed drawn from the rows every query of the block
allows, the bit test of the filter pass, the shard windows - not the kernels.  `bug` plants one of the errors the tests
must be able to catch: "seed_outside" (seed rows allowed for SOME query only), "no_bit" (the filter pass skips the bit
test), "bit0" (the shard window starts one bit late) and "word_edge" (bit 31 of a word read from the next word)."""
import numpy as np

import search_model as M


def pack(mask):
    """bool (..., N) -> uint32 words (..., ceil(N / 32)): row r = bit r & 31 of word r >> 5 (rule F1)."""
    mask = np.asarray(mask, bool)
    n = mask.shape[-1]
    w = (n + 31) // 32
    pad = np.zeros(mask.shape[:-1] + (32 * w,), bool)
    pad[..., :n] = mask
    return np.packbits(pad, axis=-1, bitorder="little").view("<u4").reshape(mask.shape[:-1] + (w,))


def window(words, bit0, n, bug=None):
    """Allow sets A_q of a shard of n rows starting at global row bit0: bool (rows of words, n) (rule F1 / F6)."""
    words = np.atleast_2d(np.asarray(words, np.uint32))
    b = bit0 + np.arange(n, dtype=np.int64)
    if bug == "bit0":
        b = b + 1
    w, s = b >> 5, (b & 31).astype(np.uint32)
    if bug == "word_edge":
        w = np.where(s == 31, w + 1, w)
    w = np.minimum(w, words.shape[1] - 1)
    return ((words[:, w] >> s) & 1).astype(bool)


def seed_rows(A, S, bug=None):
    """Rule F2: the first S rows of I = the intersection of the query block's allow sets, in row order."""
    inter = A.any(axis=0) if bug == "seed_outside" else A.all(axis=0)
    return np.nonzero(inter)[0][:S]


class FilteredShardModel(M.ShardModel):
    """One shard of a filtered search: the seed over seed_rows, candidates only where the query's bit is set.  A
    disallowed row's fast score is NaN, so that no threshold (not even -inf) admits it."""

    def __init__(self, db, offset, sample_rows, words, bug=None, **kw):
        super().__init__(db, offset, sample_rows, **kw)
        self.words, self.bug = words, bug

    def begin_seed(self, q, k, k_shard):
        n = self.db.shape[0]
        self.q, self.k, self.k_shard = q, k, k_shard
        if n == 0:
            self.cand = None
            return np.full(q.shape[0], np.inf, np.float32)
        A = window(self.words, self.offset, n, self.bug)
        A = np.broadcast_to(A, (q.shape[0], n))
        fast = M.fast_scores(q, self.db)
        self.fast = fast if self.bug == "no_bit" else np.where(A, fast, np.float32(np.nan))
        s = min(max(self.sample_rows, min(n, 4 * k)), n)
        small = n <= s
        if not small and s // 32 < k:
            s = min(n, max(s, 32 * k))
        use_gmax = (not small) and (s // 32 >= k)
        rows = seed_rows(A, s, self.bug)
        nv = rows.shape[0]
        self.n_seed = nv
        thr = np.empty(q.shape[0], np.float32)
        seed2 = np.empty(q.shape[0], np.float32)
        for i in range(q.shape[0]):
            seed = fast[i, rows]
            if use_gmax:                      # full groups of 32 gathered rows; all S valid: every group, the last clipped
                if nv == s:
                    pad = (-nv) % 32
                    seed = np.concatenate([seed, np.full(pad, -np.inf, np.float32)])
                else:
                    seed = seed[:32 * (nv // 32)]
                vals = seed.reshape(-1, 32).max(axis=1)
            else:
                vals = seed
            thr[i] = M.kth_largest(vals, k) - M.BAND          # fewer than k values: -inf
            seed2[i] = M.kth_largest(vals, k_shard) - M.BAND
        self.thr = thr
        return seed2


def filtered_search(q, db, k, words, sample_rows=64, bounds=None, peer=False, bug=None, cand_cap=None, seed=0):
    """The filtered search over shards `bounds` (default: one shard); the collective protocol (MIN of the selection
    thresholds) or, peer=True, the peer-memory one (also the MIN of the seed bounds).  -> (scores, indices)."""
    from dirb200.dist import shard_quota
    bounds = bounds or [(0, db.shape[0])]
    shards = [FilteredShardModel(db[a:b], a, sample_rows, words, bug, cand_cap=cand_cap,
                                 rng=np.random.RandomState(seed + j)) for j, (a, b) in enumerate(bounds)]
    c = shard_quota(k, [b - a for a, b in bounds]) if len(bounds) > 1 else k
    if peer:
        seed_min = np.minimum.reduce([s.begin_seed(q, k, c) for s in shards])
        sel = np.minimum.reduce([s.begin_filter(seed_min) for s in shards])
    else:
        sel = np.minimum.reduce([s.begin(q, k, c) for s in shards])
    lists = [s.finish(sel) for s in shards]
    sc = np.concatenate([l[0] for l in lists], axis=1)
    ix = np.concatenate([l[1] for l in lists], axis=1)
    out_s = np.full((q.shape[0], k), -np.inf)
    out_i = np.full((q.shape[0], k), -1, np.int64)
    for i in range(q.shape[0]):
        valid = ix[i] >= 0
        order = np.lexsort((ix[i][valid], -sc[i][valid]))[:k]
        out_s[i, :order.shape[0]] = sc[i][valid][order]
        out_i[i, :order.shape[0]] = ix[i][valid][order]
    return out_s, out_i


def exact_filtered_topk(q, db, k, words):
    """Rule F5: per query the exact top-k of its allowed rows (fp64 scores, score desc, row asc), tail (-inf, -1)."""
    A = np.broadcast_to(window(words, 0, db.shape[0]), (q.shape[0], db.shape[0]))
    out_s = np.full((q.shape[0], k), -np.inf)
    out_i = np.full((q.shape[0], k), -1, np.int64)
    for i in range(q.shape[0]):
        rows = np.nonzero(A[i])[0]
        s, j = M.exact_topk(q[i:i + 1], db[rows], k)
        m = j[0] >= 0
        out_s[i, :m.sum()] = s[0][m]
        out_i[i, :m.sum()] = rows[j[0][m]]
    return out_s, out_i
