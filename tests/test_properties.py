"""Property-based tests (hypothesis) of the host-side logic: row sharding, the descriptor store, AP from a ranked
prefix vs AP from the full score row, PIL-exact resize coefficient tables.  CPU only."""
import os
import pickle

import numpy as np
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from dirb200 import dist as ddist
from dirb200 import store as S

# derandomize: the same examples on every run (a red CPU suite must mean a code change, not a new random draw);
# explore with HYP_RANDOM=1 (fresh random draws) and HYP_SCALE=n (n times more examples)
COMMON = dict(deadline=None, derandomize=os.environ.get("HYP_RANDOM", "") == "", database=None,
              suppress_health_check=[HealthCheck.function_scoped_fixture, HealthCheck.too_slow])
_SCALE = int(os.environ.get("HYP_SCALE", "1"))        # HYP_RANDOM=1 HYP_SCALE=20: a long exploratory run


@settings(max_examples=200 * _SCALE, **COMMON)
@given(n=st.integers(0, 10**7), world=st.integers(1, 64))
def test_shard_rows_partitions_the_rows(n, world):
    rs = [ddist.shard_rows(n, world, r) for r in range(world)]
    assert rs[0][0] == 0 and rs[-1][1] == n
    assert all(a[1] == b[0] for a, b in zip(rs, rs[1:]))
    sizes = [b - a for a, b in rs]
    assert min(sizes) >= 0 and max(sizes) - min(sizes) <= 1                      # balanced to within one row


@settings(max_examples=40 * _SCALE, **COMMON)
@given(n=st.integers(0, 300), dim=st.sampled_from([1, 8, 64]), per=st.integers(1, 128), world=st.integers(1, 9),
       f16=st.booleans(), data=st.data())
def test_store_reads_equal_slices(tmp_path_factory, n, dim, per, world, f16, data):
    path = str(tmp_path_factory.mktemp("store"))
    db = np.random.RandomState(n * 31 + dim).standard_normal((n, dim)).astype(np.float32)
    stored = db.astype(np.float16) if f16 else db
    s = S.write_store(path, db, rows_per_shard=per, dtype=np.float16 if f16 else np.float32)
    assert len(s) == n and s.dim == dim and sum(x["n_rows"] for x in s.shards) == n
    a = data.draw(st.integers(0, n))
    b = data.draw(st.integers(a, n))
    assert np.array_equal(s.read_rows(a, b), stored[a:b])
    parts = [s.read_rows(*s.rank_range(r, world)) for r in range(world)]
    assert np.array_equal(np.concatenate(parts) if parts else stored[:0], stored)
    assert all(s.rank_range(r, world) == ddist.shard_rows(n, world, r) for r in range(world))


def _relevants_dataset(tmp, n, gnd):
    from dirtorch.datasets import ImageListRelevants
    names = ["im%04d" % i for i in range(n)]
    with open(os.path.join(tmp, "gnd.pkl"), "wb") as f:
        pickle.dump({"imlist": names, "qimlist": names[:len(gnd)], "gnd": gnd}, f)
    return ImageListRelevants(os.path.join(tmp, "gnd.pkl"), root=tmp)


@settings(max_examples=60 * _SCALE, **COMMON)
@given(n=st.integers(8, 120), seed=st.integers(0, 10**6), revisited=st.booleans(), data=st.data())
def test_ap_from_full_ranking_equals_ap_from_scores(tmp_path_factory, n, seed, revisited, data):
    """eval_query_AP_from_ranking over the COMPLETE ranking == eval_query_AP on the score row (distinct scores), and a
    prefix either reproduces it or says 'unknown' - never a different number."""
    r = np.random.RandomState(seed)
    idx = r.permutation(n)
    n_pos, n_junk = int(r.randint(1, 6)), int(r.randint(0, 4))
    pos, junk = [int(v) for v in idx[:n_pos]], [int(v) for v in idx[n_pos:n_pos + n_junk]]
    if revisited:
        cut = int(r.randint(0, n_pos + 1))
        g = {"bbx": (0, 0, 1, 1), "easy": pos[:cut], "hard": pos[cut:], "junk": junk}
    else:
        g = {"bbx": (0, 0, 1, 1), "ok": pos, "junk": junk}
    ds = _relevants_dataset(str(tmp_path_factory.mktemp("gt")), n, [g])
    scores = r.permutation(n).astype(np.float64) / n                             # distinct: no tie ambiguity
    order = np.argsort(-scores)
    full = ds.eval_query_AP(0, scores)
    got = ds.eval_query_AP_from_ranking(0, order)
    k = data.draw(st.integers(1, n))
    part = ds.eval_query_AP_from_ranking(0, order[:k])
    if isinstance(full, dict):
        for m in full:
            assert abs(got[m] - full[m]) < 1e-12
            assert part[m] is None or abs(part[m] - full[m]) < 1e-12
    else:
        assert abs(got - full) < 1e-12
        assert part is None or abs(part - full) < 1e-12


@settings(max_examples=25 * _SCALE, **COMMON)
@given(h=st.integers(2, 40), w=st.integers(2, 40), oh=st.integers(1, 60), ow=st.integers(1, 60), seed=st.integers(0, 999))
def test_resize_tables_reproduce_pil_for_any_size(h, w, oh, ow, seed):
    """The coefficient tables the GPU resize uses (dirb200_resize_coeffs, a host function of the library), applied
    in numpy integer arithmetic exactly as the kernels do, reproduce PIL's BILINEAR resize byte for byte."""
    from PIL import Image
    from dirb200 import ops
    img = np.random.RandomState(seed).randint(0, 256, (h, w, 3), dtype=np.uint8)
    ref = np.array(Image.fromarray(img).resize((ow, oh), Image.BILINEAR))

    def apply(a, in_size, out_size):                      # a: (in_size, ...) -> (out_size, ...), along axis 0
        bounds, kk = ops.resize_coeffs(in_size, out_size)
        out = np.empty((out_size,) + a.shape[1:], np.uint8)
        for o in range(out_size):
            x0, n = int(bounds[o, 0]), int(bounds[o, 1])
            acc = (1 << 21) + np.tensordot(kk[o, :n].astype(np.int64), a[x0:x0 + n].astype(np.int64), axes=(0, 0))
            out[o] = np.clip(acc >> 22, 0, 255)
        return out

    horiz = apply(img.transpose(1, 0, 2), w, ow).transpose(1, 0, 2)              # PIL: horizontal pass first
    got = apply(horiz, h, oh)
    assert np.array_equal(got, ref)


@settings(max_examples=60 * _SCALE, **COMMON)
@given(dim=st.sampled_from([64, 128, 512, 1024, 2048]), seed=st.integers(0, 10**6),
       kind=st.sampled_from(["gauss", "const", "sparse", "signed_const", "heavy", "tiny_tail", "subnormal_scaled"]))
def test_fp16_score_error_stays_inside_the_search_band(dim, seed, kind):
    """The exactness argument of the top-k search (search.cu) needs |fp16-path score - exact score| <= eps16 = 1.2e-3
    for unit-norm rows: operands rounded to fp16 (relative 2^-11 each, 2^-25 absolute in the subnormal range), products
    and sums in fp32.  Bound: (2*2^-11 + 2^-22) * sum|q_i d_i| <= 9.8e-4, + D * 2^-24 accumulation <= 1.2e-4 at D = 2048,
    + subnormal term <= 2^-25 * sqrt(D).  Checked here on adversarial families (constant vectors sit on one rounding
    error for every element; sparse and heavy-tailed vectors; rows whose tail is subnormal in fp16).  subnormal_scaled:
    rows of norm 2^-10, every entry subnormal in fp16, against the bound for un-normalised data that ops.Index
    documents, 1.2e-3 |q| |row| + 2^-24 sqrt(D) (|q| + |row|)."""
    r = np.random.RandomState(seed)
    n = 64

    def family(rows):
        if kind in ("gauss", "subnormal_scaled"):
            x = r.standard_normal((rows, dim))
        elif kind == "const":
            x = np.ones((rows, dim)) * r.uniform(0.5, 2.0, (rows, 1))
        elif kind == "signed_const":
            x = np.sign(r.standard_normal((rows, dim))) * r.uniform(0.5, 2.0, (rows, 1))
        elif kind == "sparse":
            x = r.standard_normal((rows, dim)) * (r.uniform(size=(rows, dim)) < 8.0 / dim)
            x[:, 0] += 1e-3
        elif kind == "heavy":
            x = r.standard_cauchy((rows, dim))
        else:                                                     # one dominant entry, the rest far below fp16's normal range
            x = r.standard_normal((rows, dim)) * 1e-6
            x[:, 0] = 1.0
        x = x.astype(np.float32)
        return x / np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True).astype(np.float32)

    q, d = family(n), family(n)
    bound = 1.2e-3
    if kind == "subnormal_scaled":
        d = (d * np.float32(2.0 ** -10)).astype(np.float32)
        qn = np.linalg.norm(q.astype(np.float64), axis=1)[:, None]
        dn = np.linalg.norm(d.astype(np.float64), axis=1)[None, :]
        bound = 1.2e-3 * qn * dn + 2.0 ** -24 * np.sqrt(dim) * (qn + dn)
    exact = q.astype(np.float64) @ d.astype(np.float64).T
    q16, d16 = q.astype(np.float16).astype(np.float32), d.astype(np.float16).astype(np.float32)
    fast = np.zeros((n, n), np.float32)
    for c in range(0, dim, 16):                                   # K = 16 slices accumulated in fp32, like the MMA
        fast += q16[:, c:c + 16] @ d16[:, c:c + 16].T
    err = np.abs(fast.astype(np.float64) - exact)
    assert (err <= bound).all(), (kind, dim, err.max())
    err = err.max()
    if kind in ("const", "signed_const") and dim == 2048:
        assert err > 1e-5                                         # the family does exercise the rounding term


def test_fp16_score_error_bound_is_nearly_attained():
    """Worst case of the bound above: every entry sits just below an fp16 rounding midpoint (relative error 2^-11, all
    of one sign), q = d.  The error reaches ~9.8e-4 - eps16 = 1.2e-3 is neither loose by much nor too small."""
    dim = 1024
    v = np.float32(2.0 ** -5 + 2.0 ** -16 - 2.0 ** -24)           # rounds DOWN to 2^-5 in fp16
    x = np.full(dim, v, np.float32)
    x[-1] = np.float32(np.sqrt(max(0.0, 1.0 - float((x[:-1].astype(np.float64) ** 2).sum()))))
    assert abs(np.linalg.norm(x.astype(np.float64)) - 1.0) < 1e-6
    assert float(np.float16(v)) == 2.0 ** -5
    exact = float(x.astype(np.float64) @ x.astype(np.float64))
    x16 = x.astype(np.float16).astype(np.float32)
    fast = np.float32(0)
    for c in range(0, dim, 16):
        fast = np.float32(fast + np.float32(x16[c:c + 16] @ x16[c:c + 16]))
    err = abs(float(fast) - exact)
    assert 9.0e-4 < err <= 1.2e-3, err


def _unit(x):
    return (x / np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True)).astype(np.float32)


@settings(max_examples=300 * _SCALE, **COMMON)
@given(n=st.integers(1, 1500), nq=st.integers(1, 5), k=st.integers(1, 40), shards=st.integers(1, 6),
       sample=st.sampled_from([32, 64, 256, 4096]), kind=st.sampled_from(["random", "duplicates", "clustered", "planted"]),
       seed=st.integers(0, 10**6), data=st.data())
def test_search_protocol_model_returns_the_exact_topk(n, nq, k, shards, sample, kind, seed, data):
    """The algorithm of search.cu + dist.py (group-max seed threshold, band filter, local k-th / ceil(k/G)-th
    selection, MIN exchange, exact re-scoring, merge), restated in NumPy (tests/search_model.py), returns exactly the
    top-k by (exact score desc, index asc) - for uneven and empty shards, exact duplicates (ties broken by index),
    rows clustered inside the band, and k larger than a shard or than the database."""
    import search_model as M
    r = np.random.RandomState(seed)
    dim = 64
    q = _unit(r.standard_normal((nq, dim)))
    if kind == "random":
        db = _unit(r.standard_normal((n, dim)))
    elif kind == "duplicates":                                     # few distinct rows, many exact copies
        base = _unit(r.standard_normal((max(1, n // 20), dim)))
        db = base[r.randint(0, base.shape[0], n)]
    elif kind == "clustered":                                      # scores packed within a fraction of the band
        db = _unit(q[0][None, :] + 2e-3 * r.standard_normal((n, dim)))
    else:                                                          # a handful of strong matches in a random crowd
        db = _unit(r.standard_normal((n, dim)))
        for j in r.randint(0, n, min(n, 8)):
            db[j] = _unit((q[r.randint(nq)] + 0.3 * r.standard_normal(dim))[None])[0]
    cuts = sorted(data.draw(st.lists(st.integers(0, n), min_size=shards - 1, max_size=shards - 1)))
    bounds = list(zip([0] + cuts, cuts + [n]))                     # arbitrary, possibly empty, row ranges
    got_s, got_i, _ = M.sharded_search(q, db, k, bounds, sample_rows=sample)
    ref_s, ref_i = M.exact_topk(q, db, k)
    assert np.array_equal(got_i, ref_i)
    assert np.array_equal(got_s, ref_s)


@settings(max_examples=300 * _SCALE, **COMMON)
@given(n=st.integers(1, 1500), nq=st.integers(1, 5), k=st.integers(1, 40), shards=st.integers(1, 8),
       sample=st.sampled_from([32, 64, 256, 4096]), kind=st.sampled_from(["random", "duplicates", "clustered", "planted", "skewed"]),
       seed=st.integers(0, 10**6), data=st.data())
def test_peer_memory_protocol_model_returns_the_exact_topk(n, nq, k, shards, sample, kind, seed, data):
    """dirb200_index_search_sharded restated in NumPy: the filter threshold of every shard is max(its own k-th seed bound,
    MIN over the shards of their k_shard-th seed bounds), a shard with fewer than k_shard rows above that threshold reports
    the threshold itself, then the usual MIN exchange / re-scoring / merge.  Exact top-k for uneven, tiny and empty shards,
    duplicates, rows clustered inside the band, and databases where one shard holds all the good rows ("skewed": the
    other shards' seed bounds are far below its own)."""
    import search_model as M
    r = np.random.RandomState(seed)
    dim = 64
    q = _unit(r.standard_normal((nq, dim)))
    if kind in ("random", "skewed"):
        db = _unit(r.standard_normal((n, dim)))
        if kind == "skewed":                                        # the first rows (one shard) are all close to the queries
            m = max(1, n // 6)
            db[:m] = _unit(q[r.randint(0, nq, m)] + 0.2 * r.standard_normal((m, dim)))
    elif kind == "duplicates":
        base = _unit(r.standard_normal((max(1, n // 20), dim)))
        db = base[r.randint(0, base.shape[0], n)]
    elif kind == "clustered":
        db = _unit(q[0][None, :] + 2e-3 * r.standard_normal((n, dim)))
    else:
        db = _unit(r.standard_normal((n, dim)))
        for j in r.randint(0, n, min(n, 8)):
            db[j] = _unit((q[r.randint(nq)] + 0.3 * r.standard_normal(dim))[None])[0]
    cuts = sorted(data.draw(st.lists(st.integers(0, n), min_size=shards - 1, max_size=shards - 1)))
    bounds = list(zip([0] + cuts, cuts + [n]))
    got_s, got_i, _, _ = M.sharded_search_peer(q, db, k, bounds, sample_rows=sample)
    ref_s, ref_i = M.exact_topk(q, db, k)
    assert np.array_equal(got_i, ref_i)
    assert np.array_equal(got_s, ref_s)


@settings(max_examples=120 * _SCALE, **COMMON)
@given(n=st.integers(200, 2500), k=st.integers(1, 30), shards=st.integers(2, 4), cap=st.sampled_from([64, 128, 512]),
       kind=st.sampled_from(["random", "clustered", "planted"]), seed=st.integers(0, 10**6))
def test_peer_memory_protocol_model_with_bounded_buffers_is_exact_or_fails_loudly(n, k, shards, cap, kind, seed):
    """Same with small candidate buffers: overflow -> tightened threshold -> re-run converges to the exact top-k or ends in
    the overflow error, also when the tightened threshold replaces one that came from the other shards."""
    import search_model as M
    r = np.random.RandomState(seed)
    q = _unit(r.standard_normal((3, 64)))
    if kind == "clustered":
        db = _unit(q[0][None, :] + 2e-3 * r.standard_normal((n, 64)))
    else:
        db = _unit(r.standard_normal((n, 64)))
        if kind == "planted":
            for j in r.randint(0, n, 8):
                db[j] = _unit((q[r.randint(3)] + 0.3 * r.standard_normal(64))[None])[0]
    cuts = [n * (j + 1) // shards for j in range(shards - 1)]
    bounds = list(zip([0] + cuts, cuts + [n]))
    try:
        got_s, got_i, _, _ = M.sharded_search_peer(q, db, k, bounds, sample_rows=32, cand_cap=cap, surv_cap=1024, seed=seed)
    except M.Overflow:
        assert kind == "clustered"
        return
    ref_s, ref_i = M.exact_topk(q, db, k)
    assert np.array_equal(got_i, ref_i) and np.array_equal(got_s, ref_s)


def test_seed_bound_exchange_cuts_the_candidates():
    """What the first exchange is for: on a G-way split the filter pass of every shard keeps ~k_shard / k of the candidates
    that its own k-th seed bound would let through (2.5 M -> 0.41 M per 1 000 queries on the 8 x 125k geometry on the GPU)."""
    import search_model as M
    r = np.random.RandomState(5)
    q, db = _unit(r.standard_normal((8, 64))), _unit(r.standard_normal((16000, 64)))
    bounds = [(i * 2000, (i + 1) * 2000) for i in range(8)]
    s_p, i_p, surv_p, cand_p = M.sharded_search_peer(q, db, 64, bounds, sample_rows=1024)
    assert np.array_equal(i_p, M.exact_topk(q, db, 64)[1])
    shards = [M.ShardModel(db[a:b], a, 1024) for a, b in bounds]
    for sh in shards:
        sh.begin(q, 64, 8)
    cand_local = sum(sum(c.shape[0] for c in sh.cand) for sh in shards)
    assert cand_p < 0.5 * cand_local, (cand_p, cand_local)


def test_search_protocol_threshold_exchange_cuts_the_rescoring_work():
    """What the MIN exchange is for: with G shards each shard re-scores ~k/G rows instead of ~k."""
    import search_model as M
    r = np.random.RandomState(3)
    q, db = _unit(r.standard_normal((8, 64))), _unit(r.standard_normal((8000, 64)))
    bounds = [(i * 1000, (i + 1) * 1000) for i in range(8)]
    _, idx, surv = M.sharded_search(q, db, 64, bounds, sample_rows=256)
    assert np.array_equal(idx, M.exact_topk(q, db, 64)[1])
    solo = sum(M.sharded_search(q, db[a:b], 64, [(0, b - a)], sample_rows=256)[2] for a, b in bounds)
    assert surv < 0.5 * solo


def test_selection_depth_accounts_for_small_and_empty_shards():
    """ceil(k / G) is NOT a valid selection depth when a shard holds fewer rows than that (found by the property test
    above): the shards then certify fewer than k rows and the exchanged threshold cuts true top-k rows.
    dist.shard_quota raises the depth until sum_g min(c, N_g) >= min(k, N)."""
    import search_model as M
    from dirb200.dist import shard_quota
    assert shard_quota(100, [125000] * 8) == 13 and shard_quota(100, [1000]) == 100
    assert shard_quota(2, [0, 2]) == 2 and shard_quota(4, [1, 1000]) == 3 and shard_quota(60, [70, 47930]) == 30
    assert shard_quota(10, [0, 0, 0]) == 4 and shard_quota(10, [3, 3, 3]) == 4   # fewer rows than k: everything is kept
    for k, sizes in ((7, [5, 0, 9, 1]), (40, [3, 3, 3, 100]), (1, [0, 5]), (1024, [10, 2000, 0])):
        c = shard_quota(k, sizes)
        assert sum(min(c, n) for n in sizes) >= min(k, sum(sizes)) and (c == 1 or c == -(-k // len(sizes)) or
                                                                         sum(min(c - 1, n) for n in sizes) < min(k, sum(sizes)))
    r = np.random.RandomState(0)
    q, db = _unit(r.standard_normal((1, 64))), _unit(r.standard_normal((2, 64)))
    ref = M.exact_topk(q, db, 2)[1]
    assert np.array_equal(M.sharded_search(q, db, 2, [(0, 0), (0, 2)])[1], ref)
    naive = M.sharded_search(q, db, 2, [(0, 0), (0, 2)], quota=1)[1]              # ceil(2 / 2) = 1
    assert not np.array_equal(naive, ref)


@settings(max_examples=120 * _SCALE, **COMMON)
@given(n=st.integers(200, 2500), k=st.integers(1, 30), shards=st.integers(1, 3), cap=st.sampled_from([64, 128, 512]),
       kind=st.sampled_from(["random", "clustered", "planted"]), seed=st.integers(0, 10**6))
def test_search_protocol_model_with_bounded_buffers_is_exact_or_fails_loudly(n, k, shards, cap, kind, seed):
    """With small candidate buffers the overflow -> tightened threshold -> re-run loop either converges to the exact
    top-k or ends in the overflow error (rows packed inside the band) - it never returns a different list."""
    import search_model as M
    r = np.random.RandomState(seed)
    q = _unit(r.standard_normal((3, 64)))
    if kind == "clustered":
        db = _unit(q[0][None, :] + 2e-3 * r.standard_normal((n, 64)))
    else:
        db = _unit(r.standard_normal((n, 64)))
        if kind == "planted":
            for j in r.randint(0, n, 8):
                db[j] = _unit((q[r.randint(3)] + 0.3 * r.standard_normal(64))[None])[0]
    cuts = [n * (j + 1) // shards for j in range(shards - 1)]
    bounds = list(zip([0] + cuts, cuts + [n]))
    try:
        got_s, got_i, _ = M.sharded_search(q, db, k, bounds, sample_rows=32, cand_cap=cap, surv_cap=1024, seed=seed)
    except M.Overflow:
        assert kind == "clustered"                                 # only rows packed inside the band may overflow
        return
    ref_s, ref_i = M.exact_topk(q, db, k)
    assert np.array_equal(got_i, ref_i) and np.array_equal(got_s, ref_s)


@settings(max_examples=100 * _SCALE, **COMMON)
@given(n=st.integers(2, 60), k=st.integers(1, 8), seed=st.integers(0, 10**6), dup=st.booleans())
def test_dba_neighbour_lists_drop_exactly_the_row_itself(n, k, seed, dup):
    """pipeline._drop_self (database-side augmentation, test_dir.py:33-34: the diagonal of the self-similarity is
    zeroed): from the exact top-(k+1) of row i against its own database, the k best rows other than i, best first."""
    from dirb200.pipeline import _drop_self
    import search_model as M
    r = np.random.RandomState(seed)
    db = _unit(r.standard_normal((n, 16)))
    if dup:
        db[r.randint(n)] = db[r.randint(n)]                       # an exact duplicate pair (may be the same row)
    kk = min(k + 1, n)
    s1, i1 = M.exact_topk(db, db, kk)
    s, i = _drop_self(s1, i1, np.arange(n), k)
    ex = M.exact_scores(db, db)
    for row in range(n):
        others = [j for j in np.lexsort((np.arange(n), -ex[row])) if j != row][:k]
        assert list(i[row][:len(others)]) == others[:i.shape[1]]
        assert row not in i[row]
        assert (i[row][len(others):] == -1).all() and (s[row][len(others):] == 0).all()      # fewer than k other rows
    assert i.shape[1] == min(k, kk)


def _split_gemm(xc, comp, prescale=1.0):
    """The arithmetic of whiten_tc (ops.cu): operands split into fp16 hi + fp16 lo (split_f16_kernel), product =
    hi*hi + hi*lo + lo*hi accumulated in fp32 (one K-concatenated wgmma GEMM); lo*lo is dropped.
    prescale: power of two applied to both operands before the split and removed from the product (round-2 fix)."""
    def split(a):
        a = a.astype(np.float32) * np.float32(prescale)
        hi = a.astype(np.float16)
        lo = (a - hi.astype(np.float32)).astype(np.float16)
        return hi.astype(np.float32), lo.astype(np.float32)
    xh, xl = split(xc)
    ch, cl = split(comp)
    return (xh @ ch.T + xh @ cl.T + xl @ ch.T) / np.float32(prescale * prescale)


def _whiten_case(dim, spread, seed):
    r = np.random.RandomState(seed)
    centre = _unit(r.standard_normal((1, dim)))
    x = _unit(centre + spread * r.standard_normal((96, dim)) / np.sqrt(dim))     # |x - centre| ~ spread
    comp = _unit(r.standard_normal((48, dim)))
    xc = (x - x.mean(0)).astype(np.float32)
    return xc, comp, xc.astype(np.float64) @ comp.astype(np.float64).T


def _row_rel(got, ref):
    return float((np.linalg.norm(got.astype(np.float64) - ref, axis=1) / np.linalg.norm(ref, axis=1)).max())


@settings(max_examples=30 * _SCALE, **COMMON)
@given(dim=st.sampled_from([64, 256, 2048]), spread=st.sampled_from([1.0, 0.5, 0.25]), seed=st.integers(0, 10**6))
def test_split_fp16_whitening_error_in_the_operating_regime(dim, spread, seed):
    """Unit-norm descriptors at distance >= 0.25 from their mean (trained descriptors: 0.5-0.9) projected on unit-norm
    components: the fp16 hi/lo scheme stays within 2e-5 of the fp64 result relative to the row norm - the bar of the
    GPU whitening tests - where ONE fp16 pass is off by ~5e-4."""
    xc, comp, ref = _whiten_case(dim, spread, seed)
    rel = _row_rel(_split_gemm(xc, comp), ref)
    assert rel < 2e-5, (dim, spread, rel)
    plain16 = xc.astype(np.float16).astype(np.float32) @ comp.astype(np.float16).astype(np.float32).T
    assert _row_rel(plain16, ref) > 5 * rel


def test_split_fp16_whitening_needs_a_prescale_for_tightly_clustered_rows():
    """Limit of the scheme as shipped (found by this emulation, not yet by a GPU test): the LOW halves of x - mean fall
    into fp16's subnormal range when |x - mean| is small, so the relative error grows like 1 / |x - mean| (1e-4 at
    0.01).  Multiplying both operands by 2^10 before the split (exact, undone in the epilogue's column scale) keeps
    the low halves normal and makes the error independent of the spread - the round-2 change to split_f16_kernel."""
    errs, fixed = [], []
    for spread in (1.0, 0.1, 0.01):
        xc, comp, ref = _whiten_case(2048, spread, 1)
        errs.append(_row_rel(_split_gemm(xc, comp), ref))
        fixed.append(_row_rel(_split_gemm(xc, comp, prescale=1024.0), ref))
    assert errs[0] < 5e-6 and errs[2] > 5e-5 and errs[2] > 10 * errs[0]          # degrades as the rows cluster
    assert max(fixed) < 5e-6                                                      # prescaled: flat
