"""GPU checks of truncated diffusion (csrc/diffusion_trunc.cu, Diffusion(truncation=True)) against
tests/diffusion_trunc_model.py: the graph weights bit for bit, each local subgraph exactly, f' bit-identical to the full
solve at m = N (both storage paths of the fused solver), the residual and dense-solve bounds and bit-identity across
query blocks at m < N, edge cases, the rule-T6 ranking and rank counts, and the command line end to end."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp
import torch

import diffusion_model as M
import diffusion_trunc_model as T
from conftest import REPO

pytestmark = pytest.mark.gpu


def _unit(X):
    return (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)


def _clustered(n, dim, seed=0):
    r = np.random.RandomState(seed)
    c = r.standard_normal((max(2, n // 50), dim))
    return _unit(c[r.randint(0, c.shape[0], n)] + 0.4 * r.standard_normal((n, dim)))


def _queries(X, nq, seed):
    r = np.random.RandomState(seed)
    return _unit(X[r.randint(0, X.shape[0], nq)] + 0.05 * np.random.RandomState(seed + 1).standard_normal((nq, X.shape[1])))


def _np(*ts):
    return [t.cpu().numpy() for t in ts]


def _host_weights(d):
    rp, col, a = _np(d.graph.row_ptr, d.graph.col, d.weights.a)
    return rp, col, a


def _lists(d, Q, depth):
    sc, idx = d.index.search(torch.nn.functional.pad(torch.from_numpy(Q).cuda(), (0, d.db.shape[1] - Q.shape[1])), depth)
    return _np(idx, sc)


def test_graph_weights_are_the_graph_bit_for_bit():
    from dirb200.diffusion import Diffusion
    X = _clustered(2000, 64)
    d = Diffusion(X, k=10, truncation=True)
    d0 = Diffusion(X, k=10)
    assert all(torch.equal(a, b) for a, b in zip(d.graph, d0.graph)) and d0.weights is None
    rp, col, a = _host_weights(d)
    u = d.weights.u.cpu().numpy()
    val = d.graph.val.cpu().numpy()
    n = rp.size - 1
    for i in range(n):
        s = 0.0
        for e in range(rp[i], rp[i + 1]):                 # sequential fp64 sum in ascending j
            s += a[e]
        assert u[i] == (1.0 / np.sqrt(s) if s > 0 else 0.0), i
    rows = np.repeat(np.arange(n), np.diff(rp))
    assert np.array_equal(val, a * (u[rows] * u[col]))


def _local(loc, q):
    """(rows, row_ptr, col, val, d, u, y) of query q from the ELL storage."""
    rows, cnt, col, val, dd, uu, y = (t[q].cpu().numpy() for t in loc)
    rp = np.concatenate([[0], np.cumsum(cnt)])
    lc = np.concatenate([col[:c, l] for l, c in enumerate(cnt)]) if cnt.sum() else np.zeros(0, np.int32)
    lv = np.concatenate([val[:c, l] for l, c in enumerate(cnt)]) if cnt.sum() else np.zeros(0)
    return rows, rp, lc, lv, dd, uu, y


@pytest.mark.parametrize("m", [1, 37, 400, 1999, 2000])
def test_local_subgraph_equals_the_model(m):
    from dirb200.diffusion import Diffusion
    X = _clustered(2000, 64, seed=1)
    Q = _queries(X, 9, 3)
    kq = min(5, m)
    d = Diffusion(X, k=10, truncation=True)
    loc = d.subgraphs(Q, m, kq=kq)
    W = _host_weights(d)
    idx, sc = _lists(d, Q, m)
    for q in range(Q.shape[0]):
        rows, rp, lc, lv, dd, uu, y = _local(loc, q)
        mrows, pos = T.region(idx[q], m)
        mrp, mcol, ma, md, mu, ms = T.subgraph(W, mrows)
        assert np.array_equal(rows, mrows) and np.array_equal(rp, mrp) and np.array_equal(lc, mcol)
        assert np.array_equal(dd, md) and np.array_equal(uu, mu) and np.array_equal(lv, ms)   # bit for bit
        my = T.seeds(idx[q], sc[q], mrows, pos, kq, 3.0)
        assert np.array_equal(y != 0, my != 0) and np.allclose(y, my, rtol=1e-15, atol=0)


def _identity(d, Q, **kw):
    f, it, res = d.solve(Q, **kw)
    for m in (d.n, d.n + 3):
        rows, ft, itt, rest = d.solve_truncated(Q, m, **kw)
        assert torch.equal(rows, torch.arange(d.n, device="cuda").expand(Q.shape[0], -1))
        assert torch.equal(ft, f) and torch.equal(itt, it) and torch.equal(rest, res)
    return f


def test_m_n_is_the_full_solve_bit_for_bit_at_5063_rows():
    from dirb200.diffusion import DEFAULTS, Diffusion
    X = _clustered(5063, 2048)                        # section 4.7's data: 162 KB of vectors, the shared-memory path
    d = Diffusion(X, k=50, truncation=True)
    _identity(d, _queries(X, 20, 7), kq=DEFAULTS["kq"], alpha=DEFAULTS["alpha"], iters=DEFAULTS["iters"], tol=0.0)


def test_m_n_is_the_full_solve_bit_for_bit_on_the_solve_setup():
    from dirb200.diffusion import Diffusion
    X = _clustered(3000, 64, seed=5)
    d = Diffusion(X, k=10, truncation=True)
    f = _identity(d, _queries(X, 70, 5), kq=5, alpha=0.9, iters=300, tol=1e-9)
    assert (f == 0).sum() > 0


def test_m_n_is_the_full_solve_bit_for_bit_from_global_memory():
    from dirb200.diffusion import Diffusion
    X = _clustered(9000, 64, seed=2)                  # 32 m = 288 KB: the vectors live in the workspace
    d = Diffusion(X, k=10, truncation=True)
    _identity(d, _queries(X, 12, 2), kq=5, alpha=0.95, iters=40, tol=1e-8)


@pytest.mark.parametrize("m", [300, 1000, 8000])       # 8000: the workspace path at m < N
def test_local_solves_within_bounds(m):
    from dirb200.diffusion import Diffusion
    X = _clustered(9000, 64, seed=4)
    Q = _queries(X, 8, 9)
    alpha, tol, iters, kq = 0.9, 1e-9, 300, 5
    d = Diffusion(X, k=10, truncation=True)
    loc = d.subgraphs(Q, m, kq=kq)
    rows, f, it, res = _np(*d.solve_truncated(Q, m, kq=kq, alpha=alpha, iters=iters, tol=tol))
    for q in range(Q.shape[0] if m < 5000 else 2):      # (the dense solves of 8000 rows take seconds each)
        lr, rp, lc, lv, _, _, y = _local(loc, q)
        assert np.array_equal(rows[q], lr)
        S = sp.csr_matrix((lv, lc.astype(np.int64), rp), shape=(m, m))
        ny = np.linalg.norm(y)
        true = M.true_residual(S, y, f[q], alpha)
        mx = int(np.diff(rp).max()) if rp[-1] else 0
        drift = 4 * it[q] * M.gamma_n(mx + 4) * (1 + alpha) ** 2 * ny / (1 - alpha)
        assert it[q] < iters and res[q] <= tol * ny
        assert true <= tol * ny + drift, (q, true, drift)
        fs = sla.solve(np.eye(m) - alpha * S.toarray(), y)
        assert np.linalg.norm(f[q] - fs) <= (true + 2 * m * M.U * (1 + alpha) * np.linalg.norm(fs)) / (1 - alpha)
        _, it_m, _ = M.cg(S, y, alpha, iters, tol)
        assert abs(int(it[q]) - int(it_m)) <= 1


def test_bit_identical_across_blocks_and_positions():
    from dirb200.diffusion import Diffusion
    X = _clustered(2500, 64, seed=6)
    Q = _queries(X, 70, 6)
    d = Diffusion(X, k=10, truncation=True)
    kw = dict(kq=5, alpha=0.95, iters=25, tol=1e-6)
    ref = d.solve_truncated(Q, 500, **kw)
    assert all(torch.equal(a, b) for a, b in zip(ref, d.solve_truncated(Q, 500, **kw)))
    for qb in (1, 7, 70):
        assert all(torch.equal(a, b) for a, b in zip(ref, d.solve_truncated(Q, 500, q_block=qb, **kw))), qb
    perm = np.random.RandomState(0).permutation(Q.shape[0])
    p = torch.from_numpy(perm).cuda()
    out = d.solve_truncated(Q[perm], 500, q_block=70, **kw)
    assert all(torch.equal(a, b[p]) for a, b in zip(out, ref))


def test_edge_cases():
    from dirb200.diffusion import Diffusion
    r = np.random.RandomState(2)
    X = _unit(np.abs(r.standard_normal((400, 64))))
    X[-1] = _unit(-np.ones((1, 64)))[0]               # nobody lists it back: an isolated row, d' = 0
    d = Diffusion(X, k=5, truncation=True)
    Q = _unit(np.concatenate([X[:3], -np.ones((1, 64))]))   # the last query: every score but one negative
    kw = dict(alpha=0.9, iters=30, tol=1e-10)
    rows, f, it, res = d.solve_truncated(Q, 1, kq=1, **kw)             # m = 1 = kq: f' = y' (S' = 0)
    y = np.maximum(_lists(d, Q, 1)[1][:, 0], 0.0) ** 3.0
    assert rows.shape == (4, 1) and np.allclose(f.cpu().numpy()[:, 0], y, rtol=1e-15, atol=0)
    rows, f, it, res = d.solve_truncated(Q, 5, kq=5, **kw)             # m = kq
    assert rows.shape == (4, 5)
    rows, f, it, res = d.solve_truncated(Q, 10 ** 6, kq=5, **kw)       # m > N: m' = N
    assert rows.shape == (4, 400)
    loc = d.subgraphs(Q, 400, kq=5)
    last = list(loc.rows[3].cpu().numpy()).index(399)
    assert float(loc.d[3, last]) == 0.0 and float(loc.u[3, last]) == 0.0
    loc = d.subgraphs(Q[3:], 3, kq=3)                  # R_q of the negative query holds the isolated row
    lr = list(loc.rows[0].cpu().numpy())
    assert 399 in lr and float(loc.d[0, lr.index(399)]) == 0.0
    _, f, it, res = d.solve_truncated(Q[3:], 3, kq=3, **kw)
    assert np.isfinite(f.cpu().numpy()).all()
    Xp = _unit(np.abs(r.standard_normal((300, 64))))
    dp = Diffusion(Xp, k=5, truncation=True)
    qz = _unit(np.concatenate([-np.ones((1, 64)), Xp[:1]]))   # query 0: every score negative -> y' = 0
    _, f, it, res = dp.solve_truncated(qz, 50, kq=4, **kw)
    assert not f[0].any() and int(it[0]) == 0 and float(res[0]) == 0.0
    assert f[1].any() and int(it[1]) > 0


def test_search_follows_rule_t6():
    from dirb200.diffusion import Diffusion
    X = _clustered(3000, 64, seed=8)
    Q = _queries(X, 9, 8)
    d = Diffusion(X, k=10, truncation=True)
    kw = dict(kq=5, alpha=0.9, iters=20, tol=0.0)
    m = 700
    rows, f, _, _ = _np(*d.solve_truncated(Q, m, **kw))
    assert (f == 0).sum() > 0                          # unreached rows of R_q sit at 0
    exact, esc = _lists(d, Q, d.n)
    for k in (1, m - 1, m, m + 1, d.n):
        sc, ix = _np(*d.search(Q, k, truncate=m, q_block=4, **kw))
        for q in range(Q.shape[0]):
            ref = T.ranking(rows[q], f[q], exact[q])[:k]
            assert np.array_equal(ix[q], ref), (q, k)
            fm = dict(zip(rows[q].tolist(), f[q].tolist()))
            n_in = min(k, m)
            assert np.array_equal(sc[q, :n_in].view(np.int64), np.array([fm[j] for j in ref[:n_in]]).view(np.int64))
            if k > m:
                assert np.array_equal(ix[q, m:], exact[q, m:k]) and np.array_equal(sc[q, m:], esc[q, m:k])


def test_topk_on_planted_ties_and_signed_zeros():
    from dirb200 import lib, ops
    r = np.random.RandomState(5)
    nq, m, k = 3, 5000, 5003
    rows = np.stack([np.sort(r.choice(20000, m, replace=False)) for _ in range(nq)]).astype(np.int64)
    f = r.choice([0.5, 0.25, 0.0, -0.0, 1e-300, -1e-300, 0.75], size=(nq, m)) * (r.rand(nq, m) < 0.5)
    f[:, ::7] = r.standard_normal((nq, len(range(0, m, 7))))
    f[2] = -0.0
    f[2, ::2] = 0.0
    lw = k
    li = np.stack([np.concatenate([r.permutation(rows[q]), np.setdiff1d(np.arange(20000), rows[q])[:lw - m]])
                   for q in range(nq)]).astype(np.int64)
    ls = r.standard_normal((nq, lw))
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (rows, f, li, ls)]
    for kk in (1, m - 1, m, k):
        ws = torch.empty(lib.raw("dirb200_diffusion_trunc_topk_workspace_bytes")(nq, m, kk), dtype=torch.uint8,
                         device="cuda")
        sc = torch.empty((nq, kk), dtype=torch.float64, device="cuda")
        ix = torch.empty((nq, kk), dtype=torch.int64, device="cuda")
        lib.call("dirb200_diffusion_trunc_topk", ops._ptr(t[0]), ops._ptr(t[1]), nq, m, ops._ptr(t[2]), ops._ptr(t[3]),
                 lw, kk, ops._ptr(ws), ops._ptr(sc), ops._ptr(ix), ops._stream())
        sc, ix = _np(sc, ix)
        for q in range(nq):
            ref = T.ranking(rows[q], f[q], li[q])[:kk]
            assert np.array_equal(ix[q], ref), (q, kk)
            o = np.lexsort((rows[q], -(f[q] + 0.0)))[:min(kk, m)]
            assert np.array_equal(sc[q, :min(kk, m)].view(np.int64), f[q, o].view(np.int64))


def test_rank_counts_inside_and_outside():
    from dirb200.diffusion import Diffusion
    X = _clustered(3000, 64, seed=9)
    Q = _queries(X, 20, 9)
    d = Diffusion(X, k=10, truncation=True)
    kw = dict(kq=5, alpha=0.9, iters=20, tol=0.0)
    m = 400
    rows, f, _, _ = _np(*d.solve_truncated(Q, m, **kw))
    exact, esc = _lists(d, Q, d.n)
    r = np.random.RandomState(1)
    counts, rows_all = [], []
    for q in range(Q.shape[0]):                       # about half the targets inside R_q, the rest anywhere
        c = np.unique(np.concatenate([r.choice(rows[q], 10, replace=False), r.choice(d.n, 10, replace=False)]))
        rows_all.append(c)
        counts.append(c.size)
    t_rows = np.concatenate(rows_all).astype(np.int64)
    t_off = np.concatenate([[0], np.cumsum(counts)])
    flags = (r.rand(t_rows.size) < 0.8).astype(np.uint8)
    inside, value, above = _np(*d.rank_counts_truncated(Q, t_off, t_rows, flags, m, **kw))
    n_in = 0
    for q in range(Q.shape[0]):
        rank = T.full_ranks(rows[q], f[q], exact[q])
        ex = dict(zip(exact[q].tolist(), esc[q].tolist()))
        fm = dict(zip(rows[q].tolist(), f[q].tolist()))
        for a in range(t_off[q], t_off[q + 1]):
            t = int(t_rows[a])
            assert bool(inside[a]) == (t in fm)
            n_in += t in fm
            assert value[a] == (fm[t] if t in fm else ex[t])
            assert above[a] == (rank[t] if flags[a] else 0), (q, t)
    assert 0 < n_in < t_rows.size


def _oxford_aps_truncated(rows, f, exact, gnd):
    from dirb200.datasets import compute_average_precision
    aps = []
    for qi, g in enumerate(gnd):
        junk = set(g["junk"])
        order = [j for j in T.ranking(rows[qi], f[qi], exact[qi]) if j not in junk]
        rank = {j: i for i, j in enumerate(order)}
        aps.append(compute_average_precision(np.sort([rank[p] for p in g["ok"]])))
    return aps


def test_dir_main_with_truncated_diffusion(tmp_path, monkeypatch):
    sys.path.insert(0, os.path.join(REPO, "tests"))
    import e2e_data
    from dirb200.pipeline import expand_descriptors
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root)
    ckpt = os.path.join(root, "ckpt.pt")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "model_options": dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)}, ckpt)
    monkeypatch.setenv("DB_ROOT", root)
    from dirtorch import test_dir
    saved = os.path.join(root, "saved")
    base = ["--dataset", "Oxford5K", "--checkpoint", ckpt, "--whiten", "", "--gpu", "0", "--threads", "2", "--detailed"]
    M_T = 6
    dif = ["--diffusion", "5", "3", "--diffusion-truncate", str(M_T)]
    res = test_dir.test_dir_main(base + dif + ["--save-feats", saved])
    res_l = test_dir.test_dir_main(base + dif + ["--load-feats", saved])
    res_a = test_dir.test_dir_main(base + dif + ["--load-feats", saved, "--aqe", "2", "1"])
    B = np.load(os.path.join(saved, "feats.bdescs.npy"))
    qpath = os.path.join(saved, "feats.qdescs.npy")
    Qd = np.load(qpath) if os.path.exists(qpath) else B[qn]
    p = dict(k=5, kq=3, gamma=3.0, alpha=0.99, iters=20, tol=0.0)
    Qa = expand_descriptors(torch.from_numpy(Qd).cuda(), db=torch.from_numpy(B).cuda(), k=2, alpha=1.0)
    from dirb200.diffusion import Diffusion
    d = Diffusion(B, k=p["k"], gamma=p["gamma"], truncation=True)
    for r, q in ((res, Qd), (res_l, Qd), (res_a, np.asarray(Qa, np.float32))):
        out, qi, _ = T.diffuse(B, q, m=M_T, **p)
        rows_g, fg = _np(*d.solve_truncated(q, M_T, kq=p["kq"], alpha=p["alpha"], iters=p["iters"], tol=p["tol"])[:2])
        exact = _lists(d, q, d.n)[0]
        assert np.array_equal(exact, qi)
        rows_m = np.stack([o[0] for o in out])
        f = np.stack([o[1] for o in out])
        assert np.array_equal(rows_g, rows_m)
        # decided as in test_dir_main_with_diffusion: inside R_q no labelled row lies within 2 delta of another row
        # unless they are tied in both; rows outside R_q are ordered by exact scores, which both share
        delta = np.abs(fg - f).max()
        for qi_, g in enumerate(gnd):
            for t in list(g["ok"]) + list(g["junk"]):
                if t not in rows_m[qi_]:
                    continue
                l = int(np.where(rows_m[qi_] == t)[0][0])
                far = np.abs(f[qi_] - f[qi_, l]) > 2 * delta
                tied = (f[qi_] == f[qi_, l]) & (fg[qi_] == fg[qi_, l])
                far[l] = True
                assert np.all(far | tied), (qi_, t, delta)
        np.testing.assert_allclose(r["APs"], _oxford_aps_truncated(rows_m, f, qi, gnd), rtol=0, atol=1e-12)
        np.testing.assert_allclose(r["APs"], _oxford_aps_truncated(rows_g, fg, qi, gnd), rtol=0, atol=1e-12)


def test_inputs_are_checked():
    from dirb200.diffusion import Diffusion
    X = _clustered(500, 64)
    Q = _queries(X, 3, 1)
    d = Diffusion(X, k=5, truncation=True)
    with pytest.raises(ValueError):                    # kq > m'
        d.solve_truncated(Q, 4, kq=5)
    with pytest.raises(ValueError):                    # kq > m' = N
        Diffusion(X[:4], k=2, truncation=True).solve_truncated(Q, 100, kq=5)
    for bad in (0, -1, 2.5):
        with pytest.raises(ValueError):
            d.solve_truncated(Q, bad, kq=1)
    with pytest.raises(ValueError):                    # truncation without the weights
        Diffusion(X, k=5).solve_truncated(Q, 100, kq=5)
    with pytest.raises(ValueError):
        Diffusion(X, k=5).search(Q, 10, kq=5, truncate=100)
