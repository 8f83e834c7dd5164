"""Exact search and counting on data at the edge of their error bounds (tests/band_data.py).  -m gpu

The planted decoys rank ~1.95e-3 above the traps on the fp16 path while every trap outranks every decoy exactly: the
searches are exact only because their band (2 eps16 = 2.4e-3) covers that gap.  Each search is also run with option
eps16 set to 0.45 x the gap the GPU itself produced, and must then return a different (wrong) list."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import band_data as B  # noqa: E402
import search_model as M  # noqa: E402
from oracle import dir_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _probe(ops, q, rows, filter_path=False):
    """fp16-path score of each row for q, as the H100 computes it: search_begin(k=1) on a one-row index returns it in
    `sel` (dense epilogue); filter_path: the row is the dominant one of 64, outside a 32-row seed sample (filter
    epilogue)."""
    qd = _t(q[None].astype(np.float32))
    out = []
    for r in rows:
        if filter_path:
            db = B.fillers(q, np.linspace(0.1, 1.0, 64), seed=1)
            db[40] = r
            idx = ops.Index(_t(db), check_norms=False)
            idx.set_option("sample_rows", 32)
        else:
            idx = ops.Index(_t(r[None]), check_norms=False)
        out.append(float(idx.search_begin(qd, 1, 1).cpu()[0]))
        idx.close()
    return np.array(out, np.float64)


def _gap(ops, q, db, dec, trp):
    """Measured fp16-path gap between the weakest decoy and the strongest trap."""
    pd, pt = _probe(ops, q, db[dec]), _probe(ops, q, db[trp])
    gap = pd.min() - pt.max()
    print("fp16-path gap decoys - traps: %.4e .. %.4e" % (gap, pd.max() - pt.min()))
    assert 1.25 * B.EPS16 < gap and pd.max() - pt.min() < 2 * B.EPS16, gap
    return gap


@pytest.mark.parametrize("D", [64, 256, 1024, 2048])
def test_fp16_path_error_on_worst_case_families(D):
    """|probe - exact| <= eps16, and |probe - RN-operand emulation| <= D 2^-23 sum|q16 r16|, which a wrong conversion
    mode (a 2^-11 relative error on some operand) would exceed."""
    ops = _ops()
    for name, (q, rows) in B.probe_families(D).items():
        dense = _probe(ops, q, rows)
        filt = _probe(ops, q, rows, filter_path=True)
        assert np.array_equal(dense, filt), (name, dense, filt)
        exact = M.exact_scores(q[None], rows)[0]
        emu = M.fast_scores(q[None], rows)[0].astype(np.float64)
        q16, r16 = q.astype(np.float16).astype(np.float64), rows.astype(np.float16).astype(np.float64)
        tol = D * 2.0 ** -23 * np.abs(q16[None] * r16).sum(axis=1)
        err = np.abs(dense - exact)
        print("fp16-path error D=%d %-12s max %.4e  (emulation %.4e, probe - emulation %.2e)"
              % (D, name, err.max(), np.abs(emu - exact).max(), np.abs(dense - emu).max()))
        assert (err <= B.EPS16).all(), (name, err)
        assert (np.abs(dense - emu) <= tol).all(), (name, dense - emu, tol)
        assert err.min() > 8.5e-4                                        # the family does reach the bound


def _search(ops, db, q, k, eps16=None, **opts):
    idx = ops.Index(_t(db), check_norms=False)
    for key, v in opts.items():
        idx.set_option(key, v)
    if eps16 is not None:
        idx.set_option("eps16", eps16)
    s, i = idx.search(_t(q[None]), k)
    st = idx.stats()
    idx.close()
    return s.cpu().numpy(), i.cpu().numpy(), st


@pytest.mark.parametrize("path", ["dense", "filter", "retry"])
def test_topk_decoys_and_traps(path):
    ops = _ops()
    D = 2048
    if path == "dense":
        db, q, info = B.topk_layout(D, 4096)
        opts = {}
    elif path == "filter":
        db, q, info = B.topk_layout(D, 20000)
        opts = {"sample_rows": 512}
    else:
        db, q, info = B.topk_layout(D, 20000, n_mid=300, seed_groups=False)
        opts = {"sample_rows": 256, "cand_cap": 256, "retries": 3}
    k = info["k"]
    rs, ri = O.topk(q[None], db, k)
    assert set(ri[0]) == set(info["trap"])
    s, i, st = _search(ops, db, q, k, **opts)
    np.testing.assert_array_equal(i, ri)
    assert np.array_equal(s, rs)
    if path == "dense":
        assert st["dense_rows"] == db.shape[0]
    elif path == "filter":
        assert st["dense_rows"] == 512 and st["retries"] == 0
    else:
        assert st["retries"] >= 1
    gap = _gap(ops, q, db, info["decoy"], info["trap"])
    s, i, _ = _search(ops, db, q, k, eps16=0.45 * gap, **opts)
    assert not np.array_equal(i, ri) and not set(i[0]) & set(info["trap"])


def _two_phase(ops, shards, q, k, c, eps16=None):
    qd = _t(q[None])
    for sh in shards:
        sh.set_option("eps16", B.EPS16 if eps16 is None else eps16)
    sels = [sh.search_begin(qd, k, c) for sh in shards]
    sel = torch.stack(sels).min(dim=0).values.contiguous()
    outs = [sh.search_finish(qd, k, sel) for sh in shards]
    ms, mi = ops.topk_merge(torch.stack([o[0] for o in outs]).contiguous(), torch.stack([o[1] for o in outs]).contiguous(), k)
    return ms.cpu().numpy(), mi.cpu().numpy()


def test_two_phase_search_decoys_and_traps_in_different_shards():
    ops = _ops()
    from dirb200.dist import shard_quota
    db, q, bounds, info = B.two_shard_layout(2048, 3000, 3000)
    k = info["k"]
    c = shard_quota(k, [b - a for a, b in bounds])
    assert c <= 8
    rs, ri = O.topk(q[None], db, k)
    assert set(ri[0]) == set(info["trap"]) | set(info["strong"])
    shards = [ops.Index(_t(db[a:b]), index_offset=a, check_norms=False) for a, b in bounds]
    ms, mi = _two_phase(ops, shards, q, k, c)
    np.testing.assert_array_equal(mi, ri)
    assert np.array_equal(ms, rs)
    gap = _gap(ops, q, db, info["decoy"], info["trap"])
    ms, mi = _two_phase(ops, shards, q, k, c, eps16=0.45 * gap)
    assert not np.array_equal(mi, ri) and not set(mi[0]) & set(info["trap"])


def test_peer_exchange_decoys_and_traps_in_different_shards():
    """The four phases over the peer-memory exchange (one process): decoy shard, trap shard, empty shard."""
    ops = _ops()
    from dirb200.dist import shard_quota
    db, q, bounds, info = B.two_shard_layout(2048, 3000, 3000, seed=1)
    bounds = bounds + [(6000, 6000)]
    k = info["k"]
    c = shard_quota(k, [b - a for a, b in bounds])
    assert c <= 8
    rs, ri = O.topk(q[None], db, k)
    dbt, qd = _t(db), _t(q[None])
    shards = [ops.Index(dbt[a:b].contiguous(), index_offset=a, check_norms=False) for a, b in bounds]
    for sh in shards:
        sh.set_option("deferred_check", 1)
    xs = [ops.Exchange(0, len(shards), r, 64, 64) for r in range(len(shards))]
    ops.Exchange.open_local(xs)
    gap = _gap(ops, q, db, info["decoy"], info["trap"])
    for eps16, want_exact in ((B.EPS16, True), (0.45 * gap, False), (B.EPS16, True)):
        for sh in shards:
            sh.set_option("eps16", eps16)
        for ph in (1, 2, 3):
            for sh, x in zip(shards, xs):
                sh.search_sharded(x, qd, k, c, phase=ph)
        res = [sh.search_sharded(x, qd, k, c, phase=4) for sh, x in zip(shards, xs)]
        for sh in shards:
            sh.check()
        for ps, pi in res:
            pi, ps = pi.cpu().numpy(), ps.cpu().numpy()
            if want_exact:
                np.testing.assert_array_equal(pi, ri)
                assert np.array_equal(ps, rs)
            else:
                assert not np.array_equal(pi, ri) and not set(pi[0]) & set(info["trap"])
    for x in xs:
        x.close()


def test_rank_counts_decoys_below_and_traps_above_a_positive():
    ops = _ops()
    D = 1024
    db, q, info = B.rank_layout(D, 6000)
    t = info["target"]
    rows = np.sort(np.array([t, info["strong"][2]], np.int64))
    offs = np.array([0, 2], np.int32)
    flags = np.ones(2, np.uint8)
    ref_s, ref_a = O.rank_counts(q[None], db, offs, rows)
    at = int(np.nonzero(rows == t)[0][0])
    assert ref_a[at] == len(info["strong"]) + len(info["trap"])              # derived by hand
    qd = _t(q[None])
    index = ops.Index(_t(db), check_norms=False)
    sc, above = index.rank_counts(qd, offs, rows, flags)
    assert np.array_equal(sc.cpu().numpy(), ref_s)
    np.testing.assert_array_equal(above.cpu().numpy(), ref_a)
    assert index.stats()["retries"] == 0                                     # no exact fallback
    # two shards: scores from the owning shard, counts add up
    half = db.shape[0] // 2
    parts = [ops.Index(_t(db[:half]), index_offset=0, check_norms=False),
             ops.Index(_t(db[half:]), index_offset=half, check_norms=False)]
    t_q = _t(np.zeros(2, np.int32))
    rows_d, flags_d = _t(rows), _t(flags)
    s_sum = parts[0].target_scores(qd, t_q, rows_d) + parts[1].target_scores(qd, t_q, rows_d)
    assert np.array_equal(s_sum.cpu().numpy(), ref_s)
    ab = sum(p.rank_count(qd, offs, rows_d, flags_d, s_sum) for p in parts)
    np.testing.assert_array_equal(ab.cpu().numpy(), ref_a)
    assert all(p.stats()["retries"] == 0 for p in parts)
    # below the planted one-sided errors: decoys counted for certain, traps never captured.  The positive is built like
    # a decoy, so its own fp16-path score then also lies above s_t + eps16 and it is counted as a row before itself:
    # rows past the bound are never compared exactly, which is why eps16 must bound every row's error.
    p_dec, p_trp = _probe(ops, q, db[info["decoy"]]), _probe(ops, q, db[info["trap"]])
    s_t = ref_s[at]
    one_sided = min((p_dec - s_t).min(), (s_t - p_trp).min())
    assert 9e-4 < one_sided < B.EPS16
    eps = 0.45 * one_sided
    self_above = int(_probe(ops, q, db[[t]])[0] > s_t + eps)
    index.set_option("eps16", eps)
    _, above2 = index.rank_counts(qd, offs, rows, flags)
    assert int(above2.cpu().numpy()[at]) == ref_a[at] + len(info["decoy"]) - len(info["trap"]) + self_above


def _count(index, q, off, thr, skip=None):
    sk = None if skip is None else _t(np.asarray(skip, np.int64))
    return index.count_ge(_t(q), _t(off.astype(np.int32)), _t(thr), sk).cpu().numpy()


def test_count_ge_at_rounding_midpoints():
    """Rows scoring exactly on m = (pred32(s) + s) / 2 or one fp64 step either side, for thresholds with even and odd
    significands, at binade edges, negative and +-0: counts equal to the hand-derived ones on every path."""
    ops = _ops()
    q, db, exact, thr = B.midpoint_data()
    sub = thr[::3].copy()
    skip_row = 11
    Q = np.stack([q, q])
    off = np.array([0, thr.shape[0], thr.shape[0] + sub.shape[0]], np.int64)
    thr_all = np.concatenate([thr, sub]).astype(np.float32)
    skip = np.array([-1, skip_row])
    want = np.concatenate([B.ge_counts_by_hand(exact, thr), B.ge_counts_by_hand(exact, sub, skip=skip_row)])
    index = ops.Index(_t(db), check_norms=False)
    np.testing.assert_array_equal(_count(index, Q, off, thr_all, skip), want)
    index.set_option("count_eps", 1e-3)                                      # every pair re-scored exactly
    np.testing.assert_array_equal(_count(index, Q, off, thr_all, skip), want)
    assert index.stats()["candidates"] > 16
    index.set_option("band_cap", 16)                                         # band overflow -> exact recount
    np.testing.assert_array_equal(_count(index, Q, off, thr_all, skip), want)
    assert index.stats()["retries"] >= 1
    total = np.zeros_like(want)
    n = db.shape[0]
    for lo, hi in ((0, 23), (23, 23), (23, n)):                              # uneven, one empty
        total += _count(ops.Index(_t(db[lo:hi]), index_offset=lo, check_norms=False), Q, off, thr_all, skip)
    np.testing.assert_array_equal(total, want)


@pytest.mark.parametrize("scale", [2.0 ** -10, 2.0 ** 7], ids=["norm1e-3", "norm128"])
def test_unnormalised_rows_with_the_documented_eps16(scale):
    """Rows of norm ~1e-3 (subnormal fp16 entries) and ~100, unit query, check_norms=False: option eps16 from the
    recipe of ops.Index gives the exact top-k; at norm 1e-3, 1.2e-3 |q| |row| alone does not."""
    ops = _ops()
    D = 2048
    db, q, info = B.topk_layout(D, 4096, scale=scale)
    k = info["k"]
    qn = float(np.linalg.norm(q.astype(np.float64)))
    rn = float(np.linalg.norm(db.astype(np.float64), axis=1).max())
    rs, ri = O.topk(q[None], db, k)
    s, i, _ = _search(ops, db, q, k, eps16=B.unnormalised_eps16(qn, rn, D))
    np.testing.assert_array_equal(i, ri)
    assert np.array_equal(s, rs)
    if scale < 1:
        s, i, _ = _search(ops, db, q, k, eps16=1.2e-3 * qn * rn)
        assert not np.array_equal(i, ri)
