"""CPU checks of the truncated-diffusion model (tests/diffusion_trunc_model.py, rules T1-T6) against a dense
restatement and a dense solve, against the full model at m = N, on the planted manifold in both directions; each
planted bug leaves a check; parameter validation, --diffusion-truncate parsing, and the new kernels build without
spills."""
import os
import re

import numpy as np
import pytest

import diffusion_model as M
import diffusion_trunc_model as T
from conftest import REPO

P = dict(k=6, kq=3, gamma=3.0, alpha=0.95, iters=200, tol=1e-12)


def _data(n=60, dim=12, seed=0):
    r = np.random.RandomState(seed)
    c = r.standard_normal((5, dim))
    X = c[r.randint(0, 5, n)] + 0.35 * r.standard_normal((n, dim))
    Q = c[r.randint(0, 5, 4)] + 0.35 * r.standard_normal((4, dim))
    nrm = lambda a: (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)
    return nrm(X), nrm(Q)


def _dense_check(X, Q, m, p=P, bug=None):
    """T1-T6 restated densely (submatrix of the dense A, renormalisation, dense solve, ranking) against the model;
    True when every part agrees."""
    n = X.shape[0]
    out, qi, qs = T.diffuse(X, Q, m=m, bug=bug, **p)
    S0 = M.exact_scores(X)
    nn = np.zeros((n, n), bool)
    for i in range(n):
        nn[i, [j for j in np.lexsort((np.arange(n), -S0[i]))[:p["k"] + 1] if j != i][:p["k"]]] = True
    A = np.where(nn & nn.T, np.maximum(S0, 0.0) ** p["gamma"], 0.0)
    ok = True
    for q, (rows, f, it, res, g, y) in enumerate(out):
        R = np.sort(qi[q, :min(m, n)])
        Aq = A[np.ix_(R, R)]
        d = Aq.sum(1)
        u = np.where(d > 0, 1 / np.sqrt(np.where(d > 0, d, 1)), 0.0)
        Sq = Aq * u[:, None] * u[None, :]
        yd = np.zeros(R.size)
        for j, s in zip(qi[q, :p["kq"]], qs[q, :p["kq"]]):
            yd[np.searchsorted(R, j)] = max(s, 0.0) ** p["gamma"]
        fd = np.linalg.solve(np.eye(R.size) - p["alpha"] * Sq, yd)
        Sm = np.zeros((R.size, R.size))
        Sm[np.repeat(np.arange(R.size), np.diff(g[0])), g[1]] = g[5]
        ok &= np.array_equal(rows, R)
        ok &= np.allclose(Sm, Sq, rtol=1e-13, atol=0) and np.allclose(y, yd, rtol=1e-14, atol=0)
        ok &= bool(np.linalg.norm(f - fd) <= 1e-8 * np.linalg.norm(fd) + 1e-300)
        # ranking: R_q by the dense solution, then the rest in exact order
        rank = T.full_ranks(rows, f, qi[q], bug)
        inr = np.isin(np.arange(n), R)
        ok &= bool(np.all(rank[inr] < R.size)) and np.array_equal(np.argsort(rank)[R.size:], qi[q][~np.isin(qi[q], R)])
        ok &= np.array_equal(np.argsort(rank)[:R.size], R[np.lexsort((R, -fd))]) or not np.all(np.diff(np.sort(fd)) > 1e-9)
    return ok


@pytest.mark.parametrize("m", [1 + 2, 10, 25, 59, 60, 200])
def test_model_agrees_with_a_dense_restatement(m):
    X, Q = _data()
    assert _dense_check(X, Q, m)


def test_model_at_m_n_is_the_full_model():
    X, Q = _data()
    n = X.shape[0]
    f_full, it_full, res_full, _ = M.diffuse(X, Q, **{k: v for k, v in P.items()})
    for m in (n, n + 5):
        out, _, _ = T.diffuse(X, Q, m=m, **P)
        for q, (rows, f, it, res, _, _) in enumerate(out):
            assert np.array_equal(rows, np.arange(n))
            assert np.array_equal(f, f_full[q]) and it == it_full[q] and res == res_full[q]


@pytest.mark.parametrize("bug", ["no_renorm", "global_degree", "outside_by_index", "outside_seeds", "list_order"])
def test_planted_bugs_leave_a_check(bug):
    X, Q = _data()
    assert _dense_check(X, Q, 25)
    assert not _dense_check(X, Q, 25, bug=bug)


def _manifold_aps(m):
    X, Q, pos = M.planted_manifold()
    p = dict(k=5, kq=3, gamma=3.0, alpha=0.99, iters=50, tol=0.0)
    out, qi, _ = T.diffuse(X, Q, m=m, **p)
    aps = []
    for q, (rows, f, _, _, _, _) in enumerate(out):
        aps.append(M.average_precision(T.ranking(rows, f, qi[q]), pos[q]))
    return np.mean(aps), X, Q, pos, p


def test_planted_manifold_truncation_in_both_directions():
    X, Q, pos = M.planted_manifold()
    n = X.shape[0]
    p = dict(k=5, kq=3, gamma=3.0, alpha=0.99, iters=50, tol=0.0)
    plain = np.mean([M.average_precision(M.ranking(M.exact_scores(X, Q)[q]), pos[q]) for q in range(len(pos))])
    f_full = M.diffuse(X, Q, **p)[0]
    full = np.mean([M.average_precision(M.ranking(f_full[q]), pos[q]) for q in range(len(pos))])
    small, _, _, _, _ = _manifold_aps(10)
    large, _, _, _, _ = _manifold_aps(n)
    # R_q of 10 rows holds only the start of the chain: the far end lies outside and keeps its plain (low) rank
    assert small < full - 0.15 and abs(small - plain) < 0.1, (small, plain, full)
    # an R_q that covers the chains keeps the gain of the full solve
    _, qi, _ = T.diffuse(X, Q, m=n, **p)
    cover = max(int(np.max([np.where(qi[q] == j)[0][0] for j in pos[q]])) + 1 for q in range(len(pos)))
    covered, _, _, _, _ = _manifold_aps(cover)
    assert covered > plain + 0.2 and abs(covered - full) < 0.05, (covered, full, cover)
    assert large == full


def test_kq_beyond_m_is_refused_by_the_model():
    X, Q = _data()
    with pytest.raises(ValueError):
        T.diffuse(X, Q, m=2, **P)


def test_parameter_validation():
    from dirb200.diffusion import check_truncate
    assert check_truncate(5) == 5 and check_truncate(5.0) == 5 and check_truncate(1) == 1
    for bad in (0, -3, 2.5, True, float("nan"), float("inf")):
        with pytest.raises((ValueError, OverflowError)):
            check_truncate(bad)


def test_truncate_argument_parsing():
    from dirb200.diffusion import DEFAULTS
    from dirb200.pipeline import diffusion_params, diffusion_truncate
    assert diffusion_truncate(1000) == 1000 and diffusion_truncate(7.0) == 7
    for bad in (0, 2.5, -1, float("nan")):
        with pytest.raises(ValueError):
            diffusion_truncate(bad)
    assert "truncate" not in diffusion_params([50, 10]) and diffusion_params([50, 10]) == DEFAULTS
    from dirtorch import test_dir
    for argv in (["--diffusion-truncate", "100"],                               # without --diffusion
                 ["--diffusion", "5", "3", "--diffusion-truncate", "0"],
                 ["--diffusion", "5", "3", "--diffusion-truncate", "2.5"],
                 ["--diffusion", "5", "3", "--diffusion-truncate", "x"]):
        with pytest.raises(SystemExit):
            test_dir.test_dir_main(["--dataset", "Oxford5K", "--checkpoint", "none"] + argv)


def test_truncated_counts_order_junk_by_inside_value_index():
    from dirb200.datasets import ImageListRelevants
    db = ImageListRelevants.__new__(ImageListRelevants)
    db.relevants = [[3, 7]]
    db.junk = [[5, 9]]
    db.get_relevants = lambda q, mode: db.relevants[q]
    db.get_junk = lambda q, mode: db.junk[q]
    rows = np.array([3, 5, 7, 9])
    # junk 5 is inside R_q with a small f', so it ranks before the outside positive 7 despite the larger value of 7;
    # junk 9 is outside with a value tied with positive 7: the lower index (7) wins
    inside = np.array([1, 1, 0, 0], bool)
    vals = np.array([0.5, 1e-9, 0.8, 0.8])
    above = np.array([0, 0, 4, 0])
    ap = db.eval_query_AP_from_truncated_counts(0, rows, inside, vals, above)
    from dirb200.datasets import compute_average_precision
    assert ap == compute_average_precision(np.array([0, 3]))     # 7: 4 rows before it, 1 junk among them


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "diffusion_trunc.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+diffusion_trunc_cu\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 8
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
