"""GPU checks of diffusion re-ranking (csrc/diffusion.cu, dirb200.diffusion) against tests/diffusion_model.py: the
graph's structure exactly and its values within a derived bound, the solve against its residual bound, a dense solve
and bit-identity across query blocks, rank counts exactly, and the command line end to end."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg as sla
import torch

import diffusion_model as M
from conftest import REPO

pytestmark = pytest.mark.gpu


def _unit(X):
    return (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)


def _data(kind, n, dim, seed=0):
    r = np.random.RandomState(seed)
    if kind == "clustered":
        c = r.standard_normal((max(2, n // 50), dim))
        X = c[r.randint(0, c.shape[0], n)] + 0.4 * r.standard_normal((n, dim))
    elif kind == "duplicates":
        X = r.standard_normal((n, dim))
        X[5:10] = X[0:5]
        X[10:14] = X[0]
    elif kind == "negative":
        X = r.standard_normal((n, dim))
        X[n // 2:] = -X[:n - n // 2] + 0.05 * r.standard_normal((n - n // 2, dim))
    elif kind == "isolated":
        X = np.abs(r.standard_normal((n, dim)))
        X[-1] = -np.ones(dim)
    else:
        X = r.standard_normal((n, dim))
    return _unit(X)


def _lists(d):
    sc, idx = d.index.search(d.db, d.k + 1)
    return idx.cpu().numpy(), sc.cpu().numpy()


def _val_bound(k):
    """|val_gpu - val_model| / |val_model|: w differs by CUDA pow's 2 ulp + numpy's 1 ulp (dw = 3 * 2^-52), the
    degree sum adds 2 gamma_k, u = 1/sqrt(d) two roundings per side and half of d's error, S two multiplies per side."""
    dw = 3 * 2.0 ** -52
    return 2 * dw + 2 * M.gamma_n(k) + 12 * M.U


def _csr(g):
    return g.row_ptr.cpu().numpy(), g.col.cpu().numpy(), g.val.cpu().numpy()


GRAPH_CASES = [("random", 1, 64, 3), ("random", 2, 64, 3), ("random", 6, 64, 5), ("random", 6, 64, 9),
               ("duplicates", 60, 64, 4), ("isolated", 80, 64, 4), ("negative", 80, 64, 5), ("clustered", 2000, 64, 10),
               ("clustered", 5063, 2048, 50)]


@pytest.mark.parametrize("kind,n,dim,k", GRAPH_CASES)
def test_graph_equals_the_model(kind, n, dim, k):
    from dirb200.diffusion import Diffusion
    X = _data(kind, n, dim)
    d = Diffusion(X, k=k, gamma=3.0)
    idx, sc = _lists(d)
    rp, col, val = _csr(d.graph)
    mrp, mcol, mval = M.graph(idx, sc, k, 3.0)
    assert np.array_equal(rp, mrp) and np.array_equal(col, mcol)
    assert rp[-1] <= n * k
    err = np.abs(val - mval)
    assert np.all(err <= _val_bound(k) * np.abs(mval)), float((err / np.maximum(np.abs(mval), 1e-300)).max())
    S = M.to_csr(rp, col, val, n)
    assert (S != S.T).nnz == 0                         # bit-exact symmetry
    if kind == "clustered" and n == 2000:              # the bound is tight enough to see fp32 weights
        _, _, bval = M.graph(idx, sc, k, 3.0, bug="pow32")
        assert np.any(np.abs(val - bval) > _val_bound(k) * np.abs(bval))
    if kind == "duplicates":
        assert any(idx[i, 0] != i for i in range(n))   # self not first in its own list
    if kind == "isolated":
        assert rp[-1] - rp[-2] == 0


def test_graph_structure_at_200k():
    from dirb200.diffusion import Diffusion
    n, k = 200_000, 10
    d = Diffusion(_data("clustered", n, 128, seed=3), k=k)
    rp, col, val = _csr(d.graph)
    assert rp[0] == 0 and np.all(np.diff(rp) >= 0) and np.all(np.diff(rp) <= k) and rp[-1] == col.size
    rows = np.repeat(np.arange(n), np.diff(rp))
    assert np.all(col != rows) and np.all((col[1:] > col[:-1]) | (rows[1:] != rows[:-1]))
    S = M.to_csr(rp, col, val, n)
    assert (S != S.T).nnz == 0
    d2 = Diffusion(d.db, k=k)
    assert all(torch.equal(a, b) for a, b in zip(d.graph, d2.graph))     # the same bits on every run


def _solve_setup(n=3000, nq=70, k=10, seed=5):
    from dirb200.diffusion import Diffusion
    X = _data("clustered", n, 64, seed=seed)
    Q = _unit(X[np.random.RandomState(seed).randint(0, n, nq)] + 0.05 * np.random.RandomState(seed + 1).standard_normal((nq, 64)))
    return Diffusion(X, k=k), Q


def test_solve_residual_dense_solve_and_iterations():
    d, Q = _solve_setup()
    alpha, tol, iters, kq = 0.9, 1e-9, 300, 5
    f, it, res = d.solve(Q, kq=kq, alpha=alpha, iters=iters, tol=tol)
    f, it, res = f.cpu().numpy(), it.cpu().numpy(), res.cpu().numpy()
    n = d.n
    rp, col, val = _csr(d.graph)
    S = M.to_csr(rp, col, val, n)
    qs, qi = d.index.search(torch.from_numpy(np.pad(Q, ((0, 0), (0, d.db.shape[1] - 64)))).cuda(), kq)
    Y = M.seeds(qi.cpu().numpy(), qs.cpu().numpy(), n, 3.0)
    m = int(np.diff(rp).max())
    lu = sla.lu_factor(np.eye(n) - alpha * S.toarray())
    _, it_m, _ = M.solve(S, Y, alpha, iters, tol)
    for q in range(Q.shape[0]):
        y = Y[:, q]
        ny = np.linalg.norm(y)
        true = M.true_residual(S, y, f[q], alpha)
        # recurrence drift: per iteration the SpMM (m + 4 terms) and the two updates round, on vectors bounded by
        # (1 + alpha) ||y|| / (1 - alpha)
        drift = 4 * it[q] * M.gamma_n(m + 4) * (1 + alpha) ** 2 * ny / (1 - alpha)
        assert it[q] < iters and res[q] <= tol * ny
        assert true <= tol * ny + drift, (q, true, tol * ny, drift)
        fs = sla.lu_solve(lu, y)
        assert np.linalg.norm(f[q] - fs) <= (true + 2 * n * M.U * (1 + alpha) * np.linalg.norm(fs)) / (1 - alpha)
        assert abs(int(it[q]) - int(it_m[q])) <= 1


def test_solve_is_bit_identical_across_blocks_and_positions():
    d, Q = _solve_setup(n=2500, nq=70)
    kw = dict(kq=5, alpha=0.95, iters=25, tol=1e-6)
    ref, it0, r0 = d.solve(Q, **kw)
    again, it1, r1 = d.solve(Q, **kw)
    assert torch.equal(ref, again) and torch.equal(it0, it1) and torch.equal(r0, r1)
    for qb in (1, 7, 70):
        f, it, r = d.solve(Q, q_block=qb, **kw)
        assert torch.equal(f, ref) and torch.equal(it, it0) and torch.equal(r, r0), qb
    perm = np.random.RandomState(0).permutation(Q.shape[0])
    f, _, _ = d.solve(Q[perm], q_block=70, **kw)
    assert torch.equal(f, ref[torch.from_numpy(perm).cuda()])


def test_zero_seed_gives_zero():
    from dirb200.diffusion import Diffusion
    X = _unit(np.abs(np.random.RandomState(2).standard_normal((300, 64))))
    d = Diffusion(X, k=5)
    q = _unit(np.concatenate([-np.ones((1, 64)), X[:1]]))          # query 0: every score negative -> y = 0
    f, it, res = d.solve(q, kq=4, alpha=0.9, iters=10, tol=1e-8)
    assert not f[0].any() and int(it[0]) == 0 and float(res[0]) == 0.0
    assert f[1].any() and int(it[1]) > 0


def _kernel_rank_count(f_nq, t_off, rows, flags):
    """dirb200_diffusion_rank_count on a hand-made f (N x Q layout)."""
    import ctypes as C
    from dirb200 import lib, ops
    n, nq = f_nq.shape
    fd = torch.from_numpy(np.ascontiguousarray(f_nq)).cuda()
    off = np.ascontiguousarray(t_off, np.int32)
    T = rows.size
    ws = torch.empty(lib.raw("dirb200_diffusion_rank_count_workspace_bytes")(nq, T), dtype=torch.uint8, device="cuda")
    sc = torch.empty(T, dtype=torch.float64, device="cuda")
    ab = torch.empty(T, dtype=torch.int64, device="cuda")
    off_d, rows_d, flags_d = (torch.from_numpy(a).cuda() for a in (off, rows, flags))   # alive until the kernels ran
    lib.call("dirb200_diffusion_rank_count", ops._ptr(fd), n, nq, off.ctypes.data_as(C.c_void_p), ops._ptr(off_d),
             ops._ptr(rows_d), ops._ptr(flags_d), T, ops._ptr(ws), ops._ptr(sc), ops._ptr(ab), ops._stream())
    return sc.cpu().numpy(), ab.cpu().numpy()


def test_rank_counts_on_planted_ties_and_signed_zeros():
    r = np.random.RandomState(4)
    n, nq = 20000, 3
    f = r.choice([0.5, 0.25, 0.0, -0.0, 1e-300, -1e-300, 0.75], size=(n, nq)) * (r.rand(n, nq) < 0.5)
    f[::7] = r.standard_normal((len(range(0, n, 7)), nq))
    t_off = np.array([0, 300, 300, 900])
    rows = np.concatenate([r.choice(n, 300, replace=False), r.choice(n, 600, replace=False)]).astype(np.int64)
    flags = (r.rand(rows.size) < 0.7).astype(np.uint8)
    sc, ab = _kernel_rank_count(f, t_off, rows, flags)
    for q in range(nq):
        s = slice(t_off[q], t_off[q + 1])
        assert np.array_equal(sc[s], f[rows[s], q])
        assert np.array_equal(ab[s], M.rank_counts(f[:, q], rows[s], flags[s])), q


def test_rank_counts_of_the_solve():
    d, Q = _solve_setup(n=3000, nq=20)
    kw = dict(kq=5, alpha=0.9, iters=20, tol=0.0)
    f, _, _ = d.solve(Q, **kw)
    f = f.cpu().numpy()
    r = np.random.RandomState(1)
    counts = r.randint(0, 40, Q.shape[0])
    t_off = np.concatenate([[0], np.cumsum(counts)])
    rows = np.concatenate([r.choice(d.n, c, replace=False) for c in counts]).astype(np.int64)
    flags = (r.rand(rows.size) < 0.8).astype(np.uint8)
    sc, ab = d.rank_counts(Q, t_off, rows, flags, **kw)
    sc, ab = sc.cpu().numpy(), ab.cpu().numpy()
    assert (f == 0).sum() > 0                                          # unreached rows sit at 0
    for q in range(Q.shape[0]):
        s = slice(t_off[q], t_off[q + 1])
        assert np.array_equal(sc[s], f[q, rows[s]])
        assert np.array_equal(ab[s], M.rank_counts(f[q], rows[s], flags[s]))


def test_planted_manifold_matches_the_model():
    from dirb200.diffusion import Diffusion
    X, Q, pos = M.planted_manifold()
    p = dict(k=5, kq=3, gamma=3.0, alpha=0.99, iters=50, tol=0.0)
    f_m, _, _, _ = M.diffuse(X, Q, **p)
    d = Diffusion(X, k=p["k"], gamma=p["gamma"])
    f, _, _ = d.solve(Q, kq=p["kq"], alpha=p["alpha"], iters=p["iters"], tol=p["tol"])
    f = f.cpu().numpy()
    ap_g = [M.average_precision(M.ranking(f[q]), pos[q]) for q in range(len(pos))]
    ap_m = [M.average_precision(M.ranking(f_m[q]), pos[q]) for q in range(len(pos))]
    np.testing.assert_allclose(ap_g, ap_m, rtol=0, atol=1e-12)
    plain = np.mean([M.average_precision(M.ranking(M.exact_scores(X, Q)[q]), pos[q]) for q in range(len(pos))])
    assert np.mean(ap_g) > plain + 0.2


def _oxford_aps(f, gnd):
    from dirb200.datasets import compute_average_precision
    aps = []
    for q, g in enumerate(gnd):
        junk = set(g["junk"])
        order = [j for j in M.ranking(f[q]) if j not in junk]
        rank = {j: i for i, j in enumerate(order)}
        aps.append(compute_average_precision(np.sort([rank[p] for p in g["ok"]])))
    return aps


def test_dir_main_with_diffusion(tmp_path, monkeypatch):
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
    dif = ["--diffusion", "5", "3"]
    res = test_dir.test_dir_main(base + dif + ["--save-feats", saved])
    res_l = test_dir.test_dir_main(base + dif + ["--load-feats", saved])
    res_a = test_dir.test_dir_main(base + dif + ["--load-feats", saved, "--aqe", "2", "1"])
    B = np.load(os.path.join(saved, "feats.bdescs.npy"))
    qpath = os.path.join(saved, "feats.qdescs.npy")
    Qd = np.load(qpath) if os.path.exists(qpath) else B[qn]
    p = dict(k=5, kq=3, gamma=3.0, alpha=0.99, iters=20, tol=0.0)
    Qa = expand_descriptors(torch.from_numpy(Qd).cuda(), db=torch.from_numpy(B).cuda(), k=2, alpha=1.0)
    from dirb200.diffusion import Diffusion
    d = Diffusion(B, k=p["k"], gamma=p["gamma"])
    for r, q in ((res, Qd), (res_l, Qd), (res_a, np.asarray(Qa, np.float32))):
        f, _, _, _ = M.diffuse(B, q, **p)
        fg = d.solve(q, kq=p["kq"], alpha=p["alpha"], iters=p["iters"], tol=p["tol"])[0].cpu().numpy()
        # The comparison is decided: no value moves by more than delta = max |f_gpu - f_model| between the two, so a
        # pair of rows further apart than 2 delta in the model is ordered the same way in both; a pair at equal f
        # must be equal in both (then the lower index wins in both).
        delta = np.abs(fg - f).max()
        for qi, g in enumerate(gnd):
            for t in list(g["ok"]) + list(g["junk"]):
                far = np.abs(f[qi] - f[qi, t]) > 2 * delta
                tied = (f[qi] == f[qi, t]) & (fg[qi] == fg[qi, t])
                far[t] = True
                assert np.all(far | tied), (qi, t, delta)
        np.testing.assert_allclose(r["APs"], _oxford_aps(f, gnd), rtol=0, atol=1e-12)
        np.testing.assert_allclose(r["APs"], _oxford_aps(fg, gnd), rtol=0, atol=1e-12)


TOPK_KS = (1, 100, 1024, 1025, 5000)


def _kernel_topk(f_nq, k):
    """dirb200_diffusion_topk on a hand-made f (N x Q layout)."""
    from dirb200 import lib, ops
    n, nq = f_nq.shape
    fd = torch.from_numpy(np.ascontiguousarray(f_nq)).cuda()
    ws = torch.empty(lib.raw("dirb200_diffusion_topk_workspace_bytes")(nq, k), dtype=torch.uint8, device="cuda")
    sc = torch.empty((nq, k), dtype=torch.float64, device="cuda")
    ix = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    lib.call("dirb200_diffusion_topk", ops._ptr(fd), n, nq, k, ops._ptr(ws), ops._ptr(sc), ops._ptr(ix), ops._stream())
    return sc.cpu().numpy(), ix.cpu().numpy()


def _check_topk(f_rows, sc, ix, k):
    for q in range(f_rows.shape[0]):
        ref = M.ranking(f_rows[q])[:k]
        assert np.array_equal(ix[q], ref), (q, k)
        assert np.array_equal(sc[q].view(np.int64), f_rows[q, ref].view(np.int64)), (q, k)   # the same bits, -0 kept


def test_topk_on_planted_ties_and_signed_zeros():
    r = np.random.RandomState(7)
    n, nq = 20000, 3
    f = r.choice([0.5, 0.25, 0.0, -0.0, 1e-300, -1e-300, 0.75], size=(n, nq)) * (r.rand(n, nq) < 0.5)
    f[::7] = r.standard_normal((len(range(0, n, 7)), nq))
    f[:, 2] = -0.0                                      # a column of signed zeros only
    f[::2, 2] = 0.0
    for k in TOPK_KS + (n,):
        sc, ix = _kernel_topk(f, k)
        _check_topk(f.T, sc, ix, k)


def test_search_equals_the_stable_argsort_of_the_solve():
    d, Q = _solve_setup(n=6000, nq=9)
    kw = dict(kq=5, alpha=0.9, iters=20, tol=0.0)
    f = d.solve(Q, **kw)[0].cpu().numpy()
    assert (f == 0).sum() > 0                                          # unreached rows sit at 0
    for k in TOPK_KS + (d.n,):
        sc, ix = d.search(Q, k, q_block=4, **kw)
        _check_topk(f, sc.cpu().numpy(), ix.cpu().numpy(), k)
    with pytest.raises(ValueError):
        d.search(Q, d.n + 1, **kw)


def test_inputs_are_checked():
    from dirb200.diffusion import graph_from_knn
    d, Q = _solve_setup(n=500, nq=3)
    with pytest.raises(ValueError):                                    # 80-d queries against 64-d rows
        d.solve(np.pad(Q, ((0, 0), (0, 16))))
    sc, idx = d.index.search(d.db, d.k + 1)
    with pytest.raises(ValueError):
        graph_from_knn(torch.where(idx == 7, torch.full_like(idx, 500), idx).contiguous(), sc, d.k, 3.0)
    with pytest.raises(ValueError):
        graph_from_knn(idx, sc, d.k - 1, 3.0)
