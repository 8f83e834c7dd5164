"""Seeded data that sits on the error bounds behind the exact search and counting kernels (numpy only).

Every value lies on a dyadic grid: unit-scale entries are multiples of 2^-26 with |x| <= 1 and norms <= 1, so every
partial sum of <q, r> is a multiple of 2^-52 of magnitude <= 1 and the fp64 score is exact in any summation order.
Rows scaled by a power of two 2^s keep the property (quantum 2^(s-26)).  exact_dot_warp, the oracle's BLAS product and
search_model.exact_scores therefore agree bit for bit, ties are real ties, and score comparisons can use ==.

Worst cases of the fp16 path (search_model.fast_scores: operands rounded to fp16, products summed in fp32):
  * every entry just below (all-down) or just above (all-up) an fp16 rounding midpoint: relative error ~2^-11 each;
  * decoys / traps for one query q: on coordinates where q rounds up, a decoy equals q, elsewhere -q; a trap is the
    mirror image.  Both round away from / towards every q_i, so the fp16-path score of a decoy overestimates its exact
    score by ~2 * 2^-11 * |q|^2 ~ 9.8e-4 and that of a trap underestimates it by as much, while their exact scores are
    both ~0.  A spare coordinate (q = 2^-5) places the exact scores: decoys <= 0, traps >= mu = 2^-20, so every trap
    outranks every decoy exactly and ranks ~1.93e-3 below them on the fp16 path - more than 1.25 * eps16, less than
    the search band 2 * eps16;
  * label-count midpoints: rows whose fp64 score is exactly m = (pred32(s) + s) / 2 or one fp64 step either side.
"""
from fractions import Fraction

import numpy as np

from label_model import boundary
from search_model import EPS16

QUANT = 2.0 ** -26          # grid of unit-scale entries
MU = 2.0 ** -20             # exact margin of the traps over the decoys (unit scale)
STEP = 2.0 ** -22           # spacing of the planted exact scores
SPARE_Q = 2.0 ** -5         # query entry of the spare coordinate (fp16-exact)


def f16_spacing(mag):
    """Spacing of the fp16 numbers at magnitude mag >= 0 (2^-24 in the subnormal range)."""
    mag = float(mag)
    if mag < 2.0 ** -14:
        return 2.0 ** -24
    return 2.0 ** (int(np.floor(np.log2(mag))) - 10)


def near_midpoint(mag, up):
    """fp32 magnitude next to the fp16 rounding midpoint just above the fp16 value at or below `mag`: 2^-9 of an fp16
    spacing above it (rounds up, away from zero) or below it (rounds down).  The error is ~half an fp16 spacing."""
    sp = f16_spacing(mag)
    lo = np.floor(float(mag) / sp) * sp
    tau = sp * 2.0 ** -9
    return lo + sp / 2 + (tau if up else -tau)


def _levels(n, budget):
    """Magnitudes of n entries, each a power of two, as large as possible with sum of squares * (1 + 2^-10)^2 <= budget:
    n_hi entries at hi, the rest at hi / 2."""
    hi = 2.0 ** -int(np.floor(np.log2(np.sqrt(n))))
    lo = hi / 2
    if n * hi * hi * (1 + 2.0 ** -10) ** 2 <= budget:
        return np.full(n, hi)
    n_hi = int(np.floor((budget / (1 + 2.0 ** -10) ** 2 - n * lo * lo) / (hi * hi - lo * lo)))
    n_hi = max(0, min(n, n_hi))
    return np.concatenate([np.full(n_hi, hi), np.full(n - n_hi, lo)])


def worst_case_vector(D, up, signs=None):
    """Norm <= 1, every entry next to an fp16 rounding midpoint (up: each rounds away from zero, else towards it)."""
    mags = np.array([near_midpoint(m, up) for m in _levels(D, 1.0)])
    x = mags if signs is None else mags * signs
    return x.astype(np.float32)


def band_query(D, seed=0):
    """-> (q (D,) fp32, up (D,) bool): body entries next to fp16 midpoints, half of each magnitude rounding up and half
    down, random signs; the last coordinate is the spare one, q = 2^-5, the one before it is 0 (so that every
    magnitude has an even count)."""
    r = np.random.RandomState(seed)
    n = D - 1
    lev = _levels(n - 1, 1.0 - SPARE_Q ** 2)
    n_hi = int((lev == lev[0]).sum())
    if n_hi % 2:
        lev[n_hi - 1] = lev[-1]
    lev = np.concatenate([lev, [0.0]])
    up = np.zeros(n, bool)
    for v in np.unique(lev[:-1]):                                # balanced within each magnitude
        idx = np.nonzero(lev == v)[0]
        up[idx[r.permutation(idx.shape[0])[: idx.shape[0] // 2]]] = True
    mags = np.array([near_midpoint(m, u) if m else 0.0 for m, u in zip(lev, up)])
    signs = np.where(r.uniform(size=n) < 0.5, -1.0, 1.0)
    q = np.concatenate([mags * signs, [SPARE_Q]]).astype(np.float32)
    return q, np.concatenate([up, [False]])


def _grid(x, scale):
    quant = QUANT * scale
    return (np.round(np.asarray(x, np.float64) / quant) * quant).astype(np.float32)


def planted_rows(q, up, kind, targets, scale=1.0, seed=0):
    """Decoys (kind 'decoy', fp16-path score above the exact one) or traps ('trap', below it) for query q, one row per
    entry of `targets`; the exact score of row j is the nearest grid value at or below (decoys) / at or above (traps)
    scale * targets[j].  Row j leaves out one pair of body coordinates (one rounding up, one down, same magnitude)
    so that no two rows are equal.  scale: a power of two; the rows' entries then sit next to the fp16 midpoints at
    that scale (subnormal midpoints for small scales)."""
    D = q.shape[0]
    body = np.arange(D - 1)
    sign_q = np.sign(q[body]).astype(np.float64)
    sign_a = np.where(up[body], sign_q, -sign_q)                 # sign of q's own fp16 rounding error
    s_row = sign_a if kind == "decoy" else -sign_a
    mags = np.array([near_midpoint(scale * abs(float(v)), u) for v, u in zip(q[body], up[body])])
    base = mags * s_row
    r = np.random.RandomState(seed + (0 if kind == "decoy" else 1))
    ups, downs = np.nonzero(up[body])[0], np.nonzero(~up[body])[0]
    out = np.zeros((len(targets), D), np.float32)
    for j, t in enumerate(targets):
        row = np.concatenate([base, [0.0]])
        i_up = ups[r.randint(ups.shape[0])]
        same = downs[np.abs(np.abs(q[downs]) / abs(q[i_up]) - 1) < 1e-2]
        row[[i_up, same[r.randint(same.shape[0])]]] = 0.0
        row = row.astype(np.float32)
        b = float(np.dot(q[:-1].astype(np.float64), row[:-1].astype(np.float64)))    # exact (grid)
        quant = QUANT * scale
        spare = (scale * t - b) / SPARE_Q / quant
        row[-1] = np.float32((np.floor(spare) if kind == "decoy" else np.ceil(spare)) * quant)
        out[j] = row
    return out


def fillers(q, alphas, scale=1.0, seed=0):
    """Rows -alpha * q (slightly perturbed, on the grid): exact scores ~ -alpha * scale, far below the decoys."""
    r = np.random.RandomState(seed)
    a = np.asarray(alphas, np.float64)[:, None]
    x = -a * q[None, :].astype(np.float64) * (1 + 0.05 * r.uniform(-1, 1, (a.shape[0], q.shape[0])))
    x /= np.maximum(1.0, np.linalg.norm(x, axis=1, keepdims=True) * (1 + 1e-6))
    return _grid(x * scale, scale)


def strong_rows(q, n, scale=1.0):
    """n rows with exact scores ~0.5 .. 0.9 (times scale): certain members of the top-k."""
    c = np.linspace(0.9, 0.5, n)[:, None]
    return _grid(c * q[None, :].astype(np.float64) * scale, scale)


def probe_families(D, seed=0):
    """Worst-case families for a probe of the fp16-path score: name -> (q (D,), rows (n, D))."""
    r = np.random.RandomState(seed)
    down = worst_case_vector(D, False)
    upv = worst_case_vector(D, True)
    signs = np.where(r.uniform(size=D) < 0.5, -1.0, 1.0)
    sc = worst_case_vector(D, False, signs)
    q, up = band_query(D, seed)
    planted = np.concatenate([planted_rows(q, up, "decoy", [0.0, -STEP], seed=seed),
                              planted_rows(q, up, "trap", [MU, MU + STEP], seed=seed)])
    return {"all_down": (down, down[None]), "all_up": (upv, upv[None]), "signed_const": (sc, sc[None]),
            "decoy_trap": (q, planted)}


def topk_layout(D, n, n_dec=16, n_trap=8, n_mid=0, seed_groups=True, scale=1.0, seed=0):
    """One query, n rows: decoys (exact <= 0), traps (exact >= MU, so k = n_trap gives exactly the traps), fillers far
    below.  seed_groups: decoy g sits at row 32 g, i.e. the first 32 n_dec rows hold one decoy per group of 32 and the
    traps lie after them; else the first 32 n_dec rows hold fillers only.  n_mid: extra fillers 6e-3 .. 2e-2 below
    the decoys (many rows above a loose seed threshold).
    -> (db (n, D), q (D,), {"decoy": rows, "trap": rows, "k": n_trap})"""
    q, up = band_query(D, seed)
    r = np.random.RandomState(seed + 11)
    dec = planted_rows(q, up, "decoy", -STEP * np.arange(n_dec), scale, seed)
    trp = planted_rows(q, up, "trap", MU + STEP * np.arange(n_trap), scale, seed)
    db = fillers(q, r.uniform(0.02, 1.0, n), scale, seed + 1)
    head = 32 * n_dec
    late = head + r.permutation(n - head)
    if seed_groups:
        pos_dec, late = 32 * np.arange(n_dec), late
    else:
        pos_dec, late = late[:n_dec], late[n_dec:]
    pos_trp, late = late[:n_trap], late[n_trap:]
    pos_mid = late[:n_mid]
    db[pos_dec], db[pos_trp] = dec, trp
    if n_mid:
        db[pos_mid] = fillers(q, r.uniform(0.006, 0.0195, n_mid), scale, seed + 2)
    return db, q, {"decoy": np.sort(pos_dec), "trap": np.sort(pos_trp), "k": n_trap}


def two_shard_layout(D, n_a, n_b, n_strong=8, n_dec=16, n_trap=4, seed=0):
    """Shard A (rows [0, n_a)): decoys + fillers.  Shard B: strong rows (exact ~0.5 .. 0.9) + traps + fillers.
    k = n_strong + n_trap: the exact top-k is B's strong rows and traps, while on the fp16 path A's decoys outrank the
    traps, and with k_shard <= min(n_strong, n_dec) the MIN over the shards' selection thresholds is A's k_shard-th
    decoy - the threshold that B's traps must survive.  -> (db, q, bounds, info)"""
    q, up = band_query(D, seed)
    r = np.random.RandomState(seed + 13)
    a = fillers(q, r.uniform(0.02, 1.0, n_a), seed=seed + 1)
    b = fillers(q, r.uniform(0.02, 1.0, n_b), seed=seed + 2)
    pos_dec = np.sort(r.choice(n_a, n_dec, replace=False))
    a[pos_dec] = planted_rows(q, up, "decoy", -STEP * np.arange(n_dec), seed=seed)
    pb = r.choice(n_b, n_strong + n_trap, replace=False)
    b[pb[:n_strong]] = strong_rows(q, n_strong)
    b[pb[n_strong:]] = planted_rows(q, up, "trap", MU + STEP * np.arange(n_trap), seed=seed)
    info = {"decoy": pos_dec, "trap": np.sort(pb[n_strong:]) + n_a, "strong": np.sort(pb[:n_strong]) + n_a,
            "k": n_strong + n_trap}
    return np.concatenate([a, b]), q, [(0, n_a), (n_a, n_a + n_b)], info


def rank_layout(D, n, n_strong=5, n_dec=7, n_trap=3, seed=0):
    """One query; a positive row with exact score in (MU/2 - 2^-31, MU/2], decoys just below it (exact <= 0) whose
    fp16-path scores lie ~9.8e-4 above it, traps just above it (exact >= MU) whose fp16-path scores lie ~9.8e-4 below,
    strong rows, fillers.  Rows ranking before the positive: the strong rows and the traps.
    -> (db, q, info) with info["target"] = the positive's row, info["strong"] = the strong rows."""
    q, up = band_query(D, seed)
    r = np.random.RandomState(seed + 17)
    db = fillers(q, r.uniform(0.02, 1.0, n), seed=seed + 1)
    pos = r.choice(n, 1 + n_strong + n_dec + n_trap, replace=False)
    p_t, p_s, p_d, p_r = pos[0], pos[1:1 + n_strong], pos[1 + n_strong:1 + n_strong + n_dec], pos[1 + n_strong + n_dec:]
    db[p_t] = planted_rows(q, up, "decoy", [MU / 2], seed=seed + 5)[0]
    db[p_s] = strong_rows(q, n_strong)
    db[p_d] = planted_rows(q, up, "decoy", -STEP * np.arange(n_dec), seed=seed)
    db[p_r] = planted_rows(q, up, "trap", MU + STEP * np.arange(n_trap), seed=seed)
    return db, q, {"target": int(p_t), "strong": np.sort(p_s), "decoy": np.sort(p_d), "trap": np.sort(p_r)}


def unnormalised_eps16(q_norm, row_norm, D):
    """Option eps16 for data that is not unit-norm: 1.2e-3 |q| |row| covers the relative fp16 roundings and the fp32
    accumulation; fp16's subnormal range rounds to an absolute 2^-25 per entry, at most 2^-25 sqrt(D) (|q| + |row|)
    over a dot product, taken twice here.  (Entries must stay below fp16's largest value, 65504.)"""
    return 1.2e-3 * q_norm * row_norm + 2.0 ** -24 * np.sqrt(D) * (q_norm + row_norm)


# ---------------------------------------------------------------------------------------------- label midpoints
# Query weights: three coordinates per level, 1, 2^-60 and 2^-120, so that a term of a score far below fp32's range
# (2^-150, 2^-203) is still an fp32-normal row entry times its weight.
MID_D = 64
_W = [1.0, 2.0 ** -60, 2.0 ** -120]


def midpoint_query():
    q = np.zeros(MID_D, np.float32)
    for lev, w in enumerate(_W):
        q[3 * lev:3 * lev + 3] = w
    return q


def _place(terms):
    """Row whose exact score with midpoint_query() is sum(terms): term j goes to coordinate j of the first level
    where term / weight is an fp32 normal (or zero) represented exactly."""
    row = np.zeros(MID_D, np.float32)
    for j, t in enumerate(terms):
        if t == 0:
            continue
        for lev, w in enumerate(_W):
            v = t / w
            if 2.0 ** -126 <= abs(v) < 2.0 ** 127 and float(np.float32(v)) == v:
                row[3 * lev + j] = np.float32(v)
                break
        else:
            raise ValueError("term %r has no exact placement" % t)
    return row


def _exact_in_any_order(terms):
    """Every partial sum of the terms (any subset) is an fp64 number: the score does not depend on the order."""
    ts = [Fraction(t) for t in terms if t != 0]
    for mask in range(1, 1 << len(ts)):
        s = sum((t for i, t in enumerate(ts) if mask >> i & 1), Fraction(0))
        if Fraction(float(s)) != s:
            return False
    return True


def midpoint_rows(s):
    """Rows scoring exactly s, pred32(s), m and the fp64 neighbours of m (m = label_model.boundary(s)).
    -> list of (label, row, exact score as a Python float)."""
    s = np.float32(s)
    pred = np.nextafter(s, np.float32(-np.inf))
    m = boundary(s)
    out = [("s", _place([float(s)]), float(s)), ("pred", _place([float(pred)]), float(pred))]
    for label, e in (("m", m), ("m-", float(np.nextafter(m, -np.inf))), ("m+", float(np.nextafter(m, np.inf)))):
        for b in (float(s), float(pred), 0.0):
            terms = [b, m - b, e - m]
            if Fraction(b) + Fraction(m - b) == Fraction(m) and Fraction(m) + Fraction(e - m) == Fraction(e) \
                    and _exact_in_any_order(terms):
                try:
                    out.append((label, _place(terms), e))
                    break
                except ValueError:
                    continue
        else:
            raise ValueError("no exact decomposition for %s of s=%r" % (label, s))
    return out


def ge_counts_by_hand(exact, thr, skip=-1):
    """count[t] = #{rows r != skip: fl32(exact[r]) >= thr[t]}, fl32 being IEEE round-to-nearest-even of the fp64 value."""
    f = np.asarray(exact, np.float64).astype(np.float32)
    keep = np.arange(f.shape[0]) != skip
    return np.array([int(((f >= np.float32(t)) & keep).sum()) for t in thr], np.int64)



def midpoint_thresholds():
    """Descending fp32 thresholds: even and odd significands, binade edges +-2^j (the spacing below differs from the
    spacing above), negative values, +0 and -0."""
    f = np.float32
    odd = lambda x, d: np.nextafter(f(x), f(d))                # noqa: E731
    return np.array([1.0, odd(0.75, 1), 0.75, 0.5, 0.3, 2.0 ** -10, odd(2.0 ** -10, 0), 0.0, -0.0, -2.0 ** -20,
                     -0.25, odd(-0.25, -1), -0.6, -1.0], np.float32)


def midpoint_data():
    """-> (q (D,), db (n, D), exact (n,) fp64 scores, thr (T,) fp32): five rows per threshold (midpoint_rows)."""
    thr = midpoint_thresholds()
    rows, exact = [], []
    for s in thr:
        for _, row, e in midpoint_rows(s):
            rows.append(row)
            exact.append(e)
    return midpoint_query(), np.stack(rows), np.array(exact, np.float64), thr
