"""Exact top-k deeper than 1024 rows: the deep finish of dirb200_index_search, query blocking under option ws_budget,
dirb200_topk_merge at G*k > 4096 and alpha-QE / alpha-DBA with thousands of neighbours.  -m gpu"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import band_data as B  # noqa: E402
import post_model as PM  # noqa: E402
import synthdata as synth  # noqa: E402
from conftest import rel_l2  # noqa: E402
from oracle import dir_oracle as O  # noqa: E402
from test_gpu_band_edges import _gap  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _assert_oracle(s, i, q, db, k):
    rs, ri = O.topk(q, db, k)
    kk = min(k, db.shape[0])
    i, s = i.cpu().numpy(), s.cpu().numpy()
    np.testing.assert_array_equal(i[:, :kk], ri)
    np.testing.assert_allclose(s[:, :kk], rs, rtol=0, atol=1e-12)
    assert (i[:, kk:] == -1).all() and (s[:, kk:] == -np.inf).all()


# n_db, n_q, dim, k, sample_rows: the small path (N <= seed sample, with a -1 tail for k > N), the filtered path with a
# group-maximum seed, the filtered path with a dense seed over all N rows (N < 32 k), D 64 / 512 / 2048, Q 1 / 70 / 1000
DEEP_CASES = [
    (3000, 70, 2048, 2999, 0), (3000, 70, 2048, 3000, 0), (3000, 70, 2048, 4000, 0),
    (200000, 4, 512, 1025, 8192), (200000, 3, 512, 5000, 4096), (200000, 1, 64, 20000, 0),
    (50000, 1000, 64, 1025, 0), (100000, 70, 2048, 2048, 0), (60000, 70, 512, 5000, 0),
]


@pytest.mark.parametrize("n_db,n_q,dim,k,sample_rows", DEEP_CASES)
def test_deep_topk_matches_oracle(n_db, n_q, dim, k, sample_rows):
    ops = _ops()
    db, q, _ = synth.make_descriptor_db(n_db, n_q, dim=dim, n_pos=10, db_seed=300 + k, q_seed=400 + k)
    index = ops.Index(_t(db))
    if sample_rows:
        index.set_option("sample_rows", sample_rows)
    s, i = index.search(_t(q), k)
    st = index.stats()
    _assert_oracle(s, i, q, db, k)
    assert st["retries"] == 0 and st["survivors"] >= n_q * min(k, n_db)
    if n_db <= 4 * k:
        assert st["dense_rows"] == n_db
    index.set_option("profile", 1)
    index.search(_t(q), k)
    prof = index.profile()
    assert prof["finish"] > 0 and prof["finish_rescore"] > 0 and prof["finish_sort"] > 0


def test_deep_prefix_matches_shallow_search():
    """The first 1024 entries of a k = 5000 search are the k = 1024 search, bit for bit."""
    ops = _ops()
    db, q, _ = synth.make_descriptor_db(100000, 70, dim=512, n_pos=10, db_seed=7, q_seed=8)
    index = ops.Index(_t(db))
    s1, i1 = index.search(_t(q), 1024)
    s5, i5 = index.search(_t(q), 5000)
    assert torch.equal(i5[:, :1024], i1)
    assert torch.equal(s5[:, :1024].view(torch.int64), s1.view(torch.int64))


def test_deep_ties_at_the_cut():
    """Identical rows straddle position 1024 and position k: lower index first, as the reference's stable order."""
    ops = _ops()
    k = 1500
    db, q, _ = synth.make_descriptor_db(20000, 3, dim=128, n_pos=0, db_seed=11, q_seed=12)
    order = np.argsort(-(q[0].astype(np.float64) @ db.T.astype(np.float64)), kind="stable")
    for pos, copies in ((1023, (5, 19990, 10000)), (k - 1, (3, 19995, 12000))):
        for c in copies:
            db[c] = db[order[pos]]
    index = ops.Index(_t(db))
    s, i = index.search(_t(q), k)
    _assert_oracle(s, i, q, db, k)
    for pos in (1023, k - 1):
        row = db[order[pos]]
        same = np.nonzero((db == row).all(axis=1))[0]
        got = [r for r in i[0].cpu().numpy() if r in set(same)]
        assert got == sorted(got) and len(same) == 4


def test_deep_band_edges():
    """Decoys and traps (tests/band_data.py) around rank k = 3000 under 2992 strong rows: exact only with the full
    band 2 eps16; with eps16 = 0.45 x the measured gap the decoys take the traps' places."""
    ops = _ops()
    D, n, n_trap, n_dec, k = 2048, 20000, 8, 16, 3000
    q, up = B.band_query(D, 0)
    r = np.random.RandomState(5)
    db = B.fillers(q, r.uniform(0.02, 1.0, n), seed=1)
    strong = B.strong_rows(q, k - n_trap)
    dec = B.planted_rows(q, up, "decoy", -B.STEP * np.arange(n_dec))
    trp = B.planted_rows(q, up, "trap", B.MU + B.STEP * np.arange(n_trap))
    pos = r.permutation(n)
    p_str, p_dec, p_trp = pos[:k - n_trap], pos[k - n_trap:k - n_trap + n_dec], pos[k - n_trap + n_dec:k + n_dec]
    db[p_str], db[p_dec], db[p_trp] = strong, dec, trp
    rs, ri = O.topk(q[None], db, k)
    assert set(p_trp) <= set(ri[0]) and not set(p_dec) & set(ri[0])
    index = ops.Index(_t(db), check_norms=False)
    s, i = index.search(_t(q[None]), k)
    np.testing.assert_array_equal(i.cpu().numpy(), ri)
    assert np.array_equal(s.cpu().numpy(), rs)
    gap = _gap(ops, q, db, p_dec, p_trp)
    index.set_option("eps16", 0.45 * gap)
    s, i = index.search(_t(q[None]), k)
    assert not np.array_equal(i.cpu().numpy(), ri) and set(p_dec) & set(i[0].cpu().numpy())


def test_deep_overflow():
    """A candidate list that overflows is refilled by the retry passes; with no retry left, or with more survivors than
    the deep finish keeps (min(2k, N)), the search raises DIRB200_EOVERFLOW instead of returning a short list."""
    ops = _ops()
    from dirb200 import lib
    k = 2000
    db, q, _ = synth.make_descriptor_db(400000, 5, dim=256, n_pos=10, db_seed=21, q_seed=22)
    index = ops.Index(_t(db))
    index.set_option("cand_cap", 1)                      # -> 2k entries, ~4k candidates: the first filter pass overflows
    index.set_option("retries", 4)
    s, i = index.search(_t(q), k)
    assert index.stats()["retries"] >= 1
    _assert_oracle(s, i, q, db, k)
    index.set_option("retries", 0)
    sc = torch.empty((5, k), dtype=torch.float64, device=DEV)
    ix = torch.empty((5, k), dtype=torch.int64, device=DEV)
    with pytest.raises(lib.DirbError) as e:
        lib.call("dirb200_index_search", index._h, _t(q).data_ptr(), 5, k, sc.data_ptr(), ix.data_ptr(), None)
    assert e.value.status == -4
    # 5000 identical rows: all of them survive, more than the 2k rounded up to whole runs = 4096 kept for k = 1025
    dup = np.repeat(db[:1], 5000, axis=0)
    idx2 = ops.Index(_t(np.vstack([dup, db[1:20000]])))
    with pytest.raises(lib.DirbError) as e:
        idx2.search(_t(db[:1]), 1025)
    assert e.value.status == -4


def test_deep_query_blocks():
    """With ws_budget below what Q queries need, dirb200_index_search runs query blocks of search_max_queries(k) and
    returns what the blocks return one by one; the two-phase API refuses such a Q."""
    ops = _ops()
    from dirb200 import lib
    k = 3000
    db, q, _ = synth.make_descriptor_db(100000, 70, dim=256, n_pos=10, db_seed=31, q_seed=32)
    index = ops.Index(_t(db))
    full = index.search_max_queries(k)
    index.set_option("ws_budget", 8 << 20)
    qb = index.search_max_queries(k)
    assert 1 <= qb < 70 and qb < full
    s, i = index.search(_t(q), k)
    _assert_oracle(s, i, q, db, k)
    parts = [index.search(_t(q[c:c + qb]), k) for c in range(0, 70, qb)]
    assert torch.equal(torch.cat([p[1] for p in parts]), i)
    assert torch.equal(torch.cat([p[0] for p in parts]).view(torch.int64), s.view(torch.int64))
    with pytest.raises(lib.DirbError) as e:
        index.search_begin(_t(q), k, k)
    assert e.value.status == -2 and "%d queries" % qb in str(e.value)
    index.search_begin(_t(q[:qb]), k, k)                 # a block that fits is accepted
    index.search_finish(_t(q[:qb]), k, torch.zeros(qb, dtype=torch.float32, device=DEV) - np.inf)


def test_deep_shards_merge_bit_identical():
    """8 shards in one process (uneven, one of 3 rows, one empty), k = 2000 (G k = 16000): begin -> MIN -> finish ->
    dirb200_topk_merge from global memory gives the single index's list bit for bit."""
    ops = _ops()
    from dirb200.dist import shard_quota
    k = 2000
    sizes = [9000, 3, 0, 7000, 5000, 6997, 6000, 6000]
    db, q, _ = synth.make_descriptor_db(sum(sizes), 9, dim=512, n_pos=10, db_seed=41, q_seed=42)
    qd = _t(q)
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    shards = [ops.Index(_t(db[a:b]), index_offset=int(a)) for a, b in zip(bounds[:-1], bounds[1:])]
    c = shard_quota(k, sizes)
    sel = torch.stack([sh.search_begin(qd, k, c) for sh in shards]).min(dim=0).values.contiguous()
    outs = [sh.search_finish(qd, k, sel) for sh in shards]
    for sh in shards:
        sh.check()
    ms, mi = ops.topk_merge(torch.stack([o[0] for o in outs]).contiguous(), torch.stack([o[1] for o in outs]).contiguous(), k)
    s, i = ops.Index(_t(db)).search(qd, k)
    assert torch.equal(mi, i)
    assert torch.equal(ms.view(torch.int64), s.view(torch.int64))
    _assert_oracle(s, i, q, db, k)


@pytest.mark.parametrize("k", [1500, 3000])
def test_deep_aqe_and_adba(k):
    """alpha-QE / alpha-DBA with k neighbours against the numpy reference of expand_descriptors, and every output
    element held to the alpha-QE bound of tests/post_model.py."""
    ops = _ops()
    from dirb200 import pipeline
    from dirb200.pipeline import expand_descriptors
    db, q, _ = synth.make_descriptor_db(8000, 8, dim=64, n_pos=10, db_seed=51, q_seed=52)
    out = expand_descriptors(q, db=db, k=k, alpha=3.0)
    assert rel_l2(out, O.expand_descriptors(q, db=db, k=k, alpha=3.0)) < 1e-5
    s, i = ops.Index(_t(db)).search(_t(q), k)
    got = ops.aqe_expand(_t(q), _t(db), i, s, 3.0)
    r, b = PM.aqe_ref(_t(q), _t(db), i, s, 3.0)
    chk = PM.check("aqe k=%d" % k, got, r, b)
    assert chk.ok, chk
    # alpha-DBA: each row's k neighbours other than itself.  The k-th score stays above 0, the reference's zeroed
    # self-similarity (8000 rows).  With thousands of small neighbour terms and no query term the fp32 sums differ
    # from the reference's by ~4e-5 (rel. L2), so the element bound is the strict check here.
    x = db
    dba = expand_descriptors(x, db=None, k=k, alpha=1.0)
    s1, i1 = ops.Index(_t(x)).search(_t(x), k + 1)
    s1, i1 = pipeline._drop_self(s1.cpu().numpy(), i1.cpu().numpy(), np.arange(x.shape[0]), k)
    nn_s, nn_i = _t(s1), _t(i1)
    got = ops.aqe_expand(_t(x), _t(x), nn_i, nn_s, 1.0)
    assert np.array_equal(got.cpu().numpy(), dba)
    r, b = PM.aqe_ref(_t(x[:100]), _t(x), nn_i[:100], nn_s[:100], 1.0)
    chk = PM.check("adba k=%d" % k, got[:100], r, b)
    assert chk.ok, chk
    assert rel_l2(dba, O.expand_descriptors(x, db=None, k=k, alpha=1.0)) < 1e-4


def test_aqe_chunks_keep_the_fmaf_order():
    """Neighbours are streamed 2048 at a time; skipped entries (-1) only shift where a chunk ends, so lists with the same
    valid neighbours in the same order give the same bits, and k <= 2048 is the single-chunk kernel."""
    ops = _ops()
    db, q, _ = synth.make_descriptor_db(8000, 6, dim=256, n_pos=10, db_seed=61, q_seed=62)
    qd, dd = _t(q), _t(db)
    s, i = ops.Index(dd).search(qd, 2500)
    pad = lambda n: (torch.full((6, n), -1, dtype=torch.int64, device=DEV), torch.zeros((6, n), dtype=torch.float64, device=DEV))
    a = ops.aqe_expand(qd, dd, i.contiguous(), s.contiguous(), 0.5)
    p1, p2 = pad(1048), pad(548)
    i2 = torch.cat([i[:, :1000], p1[0], i[:, 1000:], p2[0]], 1).contiguous()
    s2 = torch.cat([s[:, :1000], p1[1], s[:, 1000:], p2[1]], 1).contiguous()
    assert torch.equal(ops.aqe_expand(qd, dd, i2, s2, 0.5), a)
    one = ops.aqe_expand(qd, dd, i[:, :2048].contiguous(), s[:, :2048].contiguous(), 0.5)
    p = pad(2048)
    two = ops.aqe_expand(qd, dd, torch.cat([i[:, :2048], p[0]], 1).contiguous(), torch.cat([s[:, :2048], p[1]], 1).contiguous(), 0.5)
    assert torch.equal(one, two)


def test_rank_topk_deep_matches_dense_aps():
    """AP from a ranking 4096 deep equals the AP from the dense score rows."""
    _ops()
    from dirb200 import pipeline
    db_, q, pos = synth.make_descriptor_db(6000, 20, dim=128, n_pos=3000, db_seed=71, q_seed=72)

    class Ranked:                                        # AP of generic.py:196-209 from a ranking or a score row
        from_ranking = 0

        def eval_query_AP(self, qi, scores):
            return O.eval_query_ap(scores, pos[qi], [])

        def eval_query_AP_from_ranking(self, qi, ranking):
            if not np.isin(pos[qi], ranking).all():
                return None                              # a positive below the ranking: the caller scores the row
            self.from_ranking += 1
            row = np.full(db_.shape[0], -1e9)            # only the positives' ranks matter once all are in the list
            row[ranking] = -np.arange(len(ranking), dtype=np.float64)
            return self.eval_query_AP(qi, row)

    ds = Ranked()
    deep = pipeline._aps_from_topk(ds, q, db_, 4096)
    dense = [ds.eval_query_AP(qi, O.scores_exact(q[qi:qi + 1], db_)[0]) for qi in range(20)]
    np.testing.assert_allclose(deep, dense, rtol=0, atol=1e-12)
    assert ds.from_ranking > 0
