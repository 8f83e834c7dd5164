"""Filtered exact search on the GPU (DESIGN.md section 4.13, rules F1-F6).  Every result is checked against rule F5:
the unfiltered search of an index built over each query's allowed rows, with the indices mapped back, bit for bit, and
(where the sizes allow it) the numpy model of tests/filter_model.py.  -m gpu"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

import filter_model as FM

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import band_data as B  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def _unit(n, d, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn((n, d), generator=g, dtype=torch.float32)
    return (x / x.norm(dim=1, keepdim=True)).to(DEV)


def _words(ops, mask_np):
    return ops.allow_rows(torch.from_numpy(np.ascontiguousarray(mask_np)).to(DEV))


def _reference(ops, X, q, k, mask):
    """Rule F5: Index(X[A_q]).search(q, k), indices mapped back; mask (N,) shared or (Q, N) per query."""
    nq = q.shape[0]
    out_s = torch.full((nq, k), -np.inf, dtype=torch.float64, device=DEV)
    out_i = torch.full((nq, k), -1, dtype=torch.int64, device=DEV)
    groups = [(np.arange(nq), mask)] if mask.ndim == 1 else [(np.array([i]), mask[i]) for i in range(nq)]
    for qs, m in groups:
        rows = torch.from_numpy(np.nonzero(m)[0]).to(DEV)
        if rows.numel() == 0:                                # nothing allowed: all (-inf, -1)
            continue
        sub = ops.Index(X[rows].contiguous())
        s, i = sub.search(q[torch.from_numpy(qs).to(DEV)].contiguous(), k)
        sub.close()
        qi = torch.from_numpy(qs).to(DEV)
        out_s[qi] = s
        out_i[qi] = torch.where(i >= 0, rows[i.clamp(min=0)], i)
    return out_s, out_i


def _same(a, b):
    (sa, ia), (sb, ib) = a, b
    assert torch.equal(ia, ib)
    assert torch.equal(sa.view(torch.int64), sb.view(torch.int64))          # score bits


def _shared_masks(n, r):
    yield "rand50", r.rand(n) < 0.5
    yield "rand10", r.rand(n) < 0.1
    yield "rand1", r.rand(n) < 0.01
    blk = np.zeros(n, bool)
    blk[n - max(1, n // 10):] = True
    yield "block_end", blk
    one = np.zeros(n, bool)
    one[n // 2] = True
    yield "one_row", one
    yield "empty", np.zeros(n, bool)
    few = np.zeros(n, bool)
    few[r.choice(n, min(n, 5), replace=False)] = True
    yield "fewer_than_k", few


@pytest.mark.parametrize("n,d", [(1, 64), (777, 64), (50000, 64), (200000, 2048)])
def test_shared_sets(n, d):
    ops = _ops()
    X = _unit(n, d, seed=n)
    q = _unit(13, d, seed=n + 1)
    index = ops.Index(X)
    allw = _words(ops, np.ones(n, bool))
    for k in (1, 100, 1024, 5000):              # every bit set == the unfiltered search, deep path included
        _same(index.search(q, k, allow=allw), index.search(q, k))
    r = np.random.RandomState(n)
    for name, m in _shared_masks(n, r):
        w = _words(ops, m)
        for k in ((10, 100, 5000) if name == "rand50" else (10, 100)):
            got = index.search(q, k, allow=w)
            _same(got, _reference(ops, X, q, k, m))
            if n * d <= 50000 * 64 and k <= 100:
                ms, mi = FM.filtered_search(q.cpu().numpy(), X.cpu().numpy(), k, FM.pack(m), sample_rows=8192)
                assert np.array_equal(got[1].cpu().numpy(), mi), name
                gs = got[0].cpu().numpy()
                assert np.array_equal(np.isfinite(gs), np.isfinite(ms)), name
                fin = np.isfinite(ms)
                assert np.abs(gs[fin] - ms[fin]).max(initial=0) < 1e-12, name


def test_per_query_sets():
    ops = _ops()
    n, d, nq, k = 20000, 64, 12, 50
    X = _unit(n, d, seed=7)
    q = X[:nq].clone()                                       # queries = database rows
    index = ops.Index(X)
    r = np.random.RandomState(8)
    loo = np.ones((nq, n), bool)
    loo[np.arange(nq), np.arange(nq)] = False
    disj = np.zeros((nq, n), bool)
    for i in range(nq):
        disj[i, i % 3::3] = True                            # three classes: no row is allowed for every query
    cases = {"self_exclusion": loo, "random": r.rand(nq, n) < 0.3, "disjoint": disj}
    for name, m in cases.items():
        got = index.search(q, k, allow=_words(ops, m))
        _same(got, _reference(ops, X, q, k, m))
        ms, mi = FM.filtered_search(q.cpu().numpy(), X.cpu().numpy(), k, FM.pack(m), sample_rows=8192)
        assert np.array_equal(got[1].cpu().numpy(), mi), name
        if name == "self_exclusion":
            assert not (got[1].cpu().numpy() == np.arange(nq)[:, None]).any()
        if name == "disjoint":                               # I is empty: seed -inf, the retries tighten the threshold
            assert index.stats()["retries"] >= 1
    # junk lists through allow_exclude, on a shared base set
    base_m = r.rand(n) < 0.6
    junk = [r.choice(n, int(r.randint(0, 300)), replace=True) for _ in range(nq)]
    pq = ops.allow_exclude(_words(ops, base_m), nq, junk)
    m = np.repeat(base_m[None], nq, axis=0)
    for i, j in enumerate(junk):
        m[i, j] = False
    assert torch.equal(pq, _words(ops, m))
    _same(index.search(q, k, allow=pq), _reference(ops, X, q, k, m))


def test_deep_k_and_tiny_budget_blocks():
    ops = _ops()
    n, d, nq = 30000, 64, 40
    X = _unit(n, d, seed=11)
    q = _unit(nq, d, seed=12)
    r = np.random.RandomState(13)
    m = r.rand(nq, n) < 0.7
    w = _words(ops, m)
    index = ops.Index(X)
    _same(index.search(q, 2000, allow=w), _reference(ops, X, q, 2000, m))          # deep path, per-query sets
    want = index.search(q, 10, allow=w)
    index.set_option("sample_rows", 1024)
    index.set_option("ws_budget", 200_000)                  # several query blocks, each with its own seed rows
    assert 1 < index.search_max_queries(10) < nq
    got = index.search(q, 10, allow=w)
    _same(got, want)
    _same(got, index.search(q, 10, allow=w))                # two runs bit-identical
    index.set_option("ws_budget", 100_000)                   # the seed buffer alone does not fit: refused
    from dirb200.lib import DirbError
    with pytest.raises(DirbError) as e:
        index.search(q[:1].contiguous(), 10, allow=w[:1].contiguous())
    assert e.value.status == -2


def test_candidate_cap_retry_overflow_and_fallback():
    ops = _ops()
    from dirb200 import lib
    from dirb200.lib import DirbError
    n, d, nq, k = 60000, 256, 5, 50
    X = _unit(n, d, seed=21)
    q = _unit(nq, d, seed=22)
    m = np.random.RandomState(23).rand(n) < 0.5
    w = _words(ops, m)
    want = _reference(ops, X, q, k, m)
    index = ops.Index(X)
    index.set_option("sample_rows", 256)
    index.set_option("cand_cap", 512)
    index.set_option("retries", 3)
    _same(index.search(q, k, allow=w), want)
    assert index.stats()["retries"] >= 1
    index.set_option("retries", 0)
    sc = torch.empty((nq, k), dtype=torch.float64, device=DEV)
    ix = torch.empty((nq, k), dtype=torch.int64, device=DEV)
    lib.call("dirb200_index_set_allow", index._h, C.c_void_p(w.data_ptr()), 0, 0)
    try:
        with pytest.raises(DirbError) as e:
            lib.call("dirb200_index_search", index._h, C.c_void_p(q.data_ptr()), nq, k, C.c_void_p(sc.data_ptr()),
                     C.c_void_p(ix.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert e.value.status == -4
    finally:
        lib.call("dirb200_index_set_allow", index._h, None, 0, 0)
    index.set_option("sample_rows", 256)
    index.set_option("cand_cap", 512)
    index.set_option("retries", 0)
    _same(index.search(q, k, allow=w), want)                 # the Python fallback re-runs with more retries


@pytest.mark.parametrize("inside", [True, False])
def test_band_decoys_inside_and_outside(inside):
    ops = _ops()
    D = 2048
    db, qv, info = B.topk_layout(D, 20000)
    X = torch.from_numpy(db).to(DEV)
    q = torch.from_numpy(qv[None]).to(DEV)
    m = np.ones(db.shape[0], bool)
    m[info["trap"][::2]] = False                             # half of the true top-k is not allowed
    if not inside:
        m[info["decoy"]] = False
    k = info["k"]
    index = ops.Index(X)
    index.set_option("sample_rows", 512)
    got = index.search(q, k, allow=_words(ops, m))
    _same(got, _reference(ops, X, q, k, m))
    gi = set(got[1].cpu().numpy()[0].tolist())
    assert gi & set(info["trap"][1::2]) == set(info["trap"][1::2])
    assert not gi & set(info["trap"][::2])


def _shards(ops, X, sizes):
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    shards = [ops.Index(X[a:b].contiguous(), index_offset=int(a)) for a, b in zip(bounds[:-1], bounds[1:])]
    for sh in shards:
        sh.n_global = int(bounds[-1])                         # allow sets number the rows of the whole database
    return shards


@pytest.mark.parametrize("sizes", [(1000, 0, 37, 5000, 2963), (4001, 3333, 1666), (700, 1, 1299, 2500, 77, 3000, 423, 2000)],
                         ids=lambda z: "-".join(map(str, z)))
def test_shards_collective_and_peer(sizes):
    ops = _ops()
    from dirb200.dist import ShardedIndex, shard_quota
    n, d, nq, k = sum(sizes), 128, 24, 50
    X = _unit(n, d, seed=31)
    q = _unit(nq, d, seed=32)
    r = np.random.RandomState(33)
    shared = r.rand(n) < 0.2
    shared[sizes[0]:sizes[0] + sizes[1] + sizes[2]] = False   # shards 1 and 2 allow nothing
    perq = r.rand(nq, n) < 0.5
    perq[:, :sizes[0]] &= (np.arange(sizes[0]) % 7 == 0)      # uneven allowed counts
    one = ops.Index(X)
    c = shard_quota(k, list(sizes))
    G = len(sizes)
    for m in (shared, perq):
        w = _words(ops, m)
        want = one.search(q, k, allow=w)
        _same(want, _reference(ops, X, q, k, m))
        shards = _shards(ops, X, sizes)
        sels = [sh.search_begin(q, k, c, allow=w) for sh in shards]          # collective: MIN of sel, finish, merge
        sel = torch.stack(sels).min(dim=0).values.contiguous()
        outs = [sh.search_finish(q, k, sel) for sh in shards]
        got = ops.topk_merge(torch.stack([o[0] for o in outs]).contiguous(), torch.stack([o[1] for o in outs]).contiguous(), k)
        _same(got, want)
        xs = [ops.Exchange(0, G, g, 64, 64) for g in range(G)]               # peer memory: the four phases shard by shard
        ops.Exchange.open_local(xs)
        for sh in shards:
            sh.set_option("deferred_check", 1)
        for _ in range(2):
            for ph in (1, 2, 3):
                for sh, x in zip(shards, xs):
                    sh.search_sharded(x, q, k, c, phase=ph, allow=w)
            res = [sh.search_sharded(x, q, k, c, phase=4) for sh, x in zip(shards, xs)]
            for sh in shards:
                sh.check()
            for got in res:
                _same(got, want)
        for x in xs:
            x.close_peers()
        for x in xs:
            x.close()
    si = ShardedIndex(X, 0)                                   # a world of one: the local filtered search
    _same(si.search(q, k, allow=_words(ops, shared)), one.search(q, k, allow=_words(ops, shared)))


def test_filter_state_and_arguments():
    ops = _ops()
    from dirb200 import lib
    from dirb200.lib import DirbError
    n, d, nq = 3000, 64, 4
    X = _unit(n, d, seed=41)
    q = _unit(nq, d, seed=42)
    m = np.random.RandomState(43).rand(n) < 0.3
    w = _words(ops, m)
    index = ops.Index(X)
    index.search(q, 20, allow=w)
    fresh = ops.Index(X)
    _same(index.search(q, 20), fresh.search(q, 20))           # the filter is gone after the call
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda t: C.c_void_p(t.data_ptr())                    # noqa: E731
    t_q = torch.zeros(1, dtype=torch.int32, device=DEV)
    t_rows = torch.zeros(1, dtype=torch.int64, device=DEV)
    t_sc = torch.zeros(1, dtype=torch.float64, device=DEV)
    off_h = np.array([0, 1, 1, 1, 1], np.int32)
    off_d = torch.from_numpy(off_h).to(DEV)
    flags = torch.ones(1, dtype=torch.uint8, device=DEV)
    above = torch.zeros(1, dtype=torch.int64, device=DEV)
    thr = torch.zeros(1, dtype=torch.float32, device=DEV)
    lab = torch.zeros(nq, dtype=torch.int64, device=DEV)
    sc = torch.zeros(nq, dtype=torch.float64, device=DEV)
    probes = torch.zeros((nq, 1), dtype=torch.int64, device=DEV)
    out_s = torch.zeros((nq, 5), dtype=torch.float64, device=DEV)
    out_i = torch.zeros((nq, 5), dtype=torch.int64, device=DEV)
    total = C.c_int64()
    calls = {
        "target_scores": ("dirb200_index_target_scores", P(q), nq, P(t_q), P(t_rows), 1, P(t_sc), stream),
        "rank_count": ("dirb200_index_rank_count", P(q), nq, off_h.ctypes.data_as(C.c_void_p), P(off_d), P(t_rows), P(flags),
                       P(t_sc), 1, P(above), stream),
        "count_ge": ("dirb200_index_count_ge", P(q), nq, P(off_d), P(thr), 1, None, P(above), stream),
        "range_search": ("dirb200_index_range_search", P(q), nq, 0.5, C.byref(total), stream),
        "self_join": ("dirb200_index_self_join", 0, n, 0.9, C.byref(total), stream),
        "nearest": ("dirb200_index_nearest", P(q), nq, P(lab), P(sc), stream),
        "search_lists": ("dirb200_index_search_lists", P(q), nq, 5, P(probes), 1, P(out_s), P(out_i), stream),
    }
    lib.call("dirb200_index_set_allow", index._h, P(w), 0, 0)
    try:
        for name, (fn, *args) in calls.items():
            with pytest.raises(DirbError) as e:
                lib.call(fn, index._h, *args)
            assert e.value.status == -5, name
    finally:
        lib.call("dirb200_index_set_allow", index._h, None, 0, 0)
    index.nearest(q)                                          # detached: the other entry points run again
    index.range_search(q, 0.5)
    for bad in (w.to(torch.int64), w.cpu(), w[:-1].contiguous(), _words(ops, np.ones((nq + 1, n), bool)),
                _words(ops, np.ones(n + 32, bool)), w.view(1, -1).expand(nq, -1)):
        with pytest.raises(ValueError):
            index.search(q, 20, allow=bad)
    with pytest.raises(ValueError):
        ops.allow_exclude(w, nq, [[n + 5000]] * nq)            # row outside the bitmap
    with pytest.raises(ValueError):
        ops.allow_exclude(w, nq, [[1]] * (nq - 1))
