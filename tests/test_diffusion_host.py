"""CPU checks of the diffusion model (tests/diffusion_model.py) against a dense restatement of the rules and a dense
linear solve; each planted bug leaves a check; parameter validation, --diffusion parsing, the planted-manifold gain,
and the kernels build without spills."""
import os
import re

import numpy as np
import pytest

import diffusion_model as M
from conftest import REPO


def _dense_S(X, k, gamma):
    """Rules 1-3 restated with dense matrices: -> (mutual mask, S)."""
    n = X.shape[0]
    S0 = M.exact_scores(X)
    nn = np.zeros((n, n), bool)
    for i in range(n):
        order = [j for j in np.lexsort((np.arange(n), -S0[i]))[:k + 1] if j != i][:k]
        nn[i, order] = True
    mut = nn & nn.T
    A = np.where(mut, np.maximum(S0, 0.0) ** gamma, 0.0)
    d = A.sum(1)
    u = np.where(d > 0, 1 / np.sqrt(np.where(d > 0, d, 1)), 0.0)
    return mut, A * u[:, None] * u[None, :]


def _data(kind, n=40, dim=12, seed=0):
    r = np.random.RandomState(seed)
    if kind == "clustered":
        c = r.standard_normal((4, dim))
        X = c[r.randint(0, 4, n)] + 0.3 * r.standard_normal((n, dim))
    elif kind == "duplicates":                       # rows 0..4 repeated: self need not come first in its list
        X = r.standard_normal((n, dim))
        X[5:10] = X[0:5]
        X[10:13] = X[0]
    elif kind == "negative":                         # anti-podal pairs: many negative scores
        X = r.standard_normal((n, dim))
        X[n // 2:] = -X[:n - n // 2] + 0.05 * r.standard_normal((n - n // 2, dim))
    else:
        X = r.standard_normal((n, dim))
    return (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)


def _model_graph(X, k, gamma, bug=None):
    idx, sc = M.topk_lists(M.exact_scores(X), k + 1)
    return M.graph(idx, sc, k, gamma, bug)


def _agrees(X, k, gamma, g):
    mut, S = _dense_S(X, k, gamma)
    n = X.shape[0]
    Sm = M.to_csr(*g, n).toarray()
    pattern = np.zeros((n, n), bool)                  # the stored entries, explicit zeros (w = 0) included
    pattern[np.repeat(np.arange(n), np.diff(g[0])), g[1]] = True
    structure = np.array_equal(pattern, mut) and g[0][-1] == mut.sum()
    return structure and np.allclose(Sm, S, rtol=1e-13, atol=0)


@pytest.mark.parametrize("kind,n,k", [("random", 40, 5), ("clustered", 40, 6), ("duplicates", 40, 4),
                                      ("negative", 30, 5), ("random", 1, 3), ("random", 2, 3), ("random", 6, 5),
                                      ("random", 6, 9)])
def test_graph_matches_dense_restatement(kind, n, k):
    X = _data(kind, n=n)
    g = _model_graph(X, k, 3.0)
    assert _agrees(X, k, 3.0, g)
    assert np.all(np.diff(g[1][g[0][0]:g[0][1]]) > 0) if g[0][1] > 1 else True
    S = M.to_csr(*g, n).toarray()
    assert np.array_equal(S, S.T)                     # bit-exact symmetry
    assert g[0][-1] <= n * k


def test_isolated_rows_have_empty_rows():
    X = _data("clustered", n=40)
    X = np.concatenate([X, -X[:1]])                  # far from everything: nobody lists it back
    g = _model_graph(X, 3, 3.0)
    assert g[0][-1] - g[0][-2] == 0
    assert _agrees(X, 3, 3.0, g)


@pytest.mark.parametrize("bug,kind", [("union", "clustered"), ("self_by_position", "duplicates"), ("dinv", "clustered")])
def test_planted_graph_bugs_leave_the_dense_restatement(bug, kind):
    X = _data(kind)
    assert _agrees(X, 5, 3.0, _model_graph(X, 5, 3.0))
    assert not _agrees(X, 5, 3.0, _model_graph(X, 5, 3.0, bug))


def test_asymmetric_product_order_breaks_bitwise_symmetry():
    X = _data("random", n=200, dim=16)
    S = M.to_csr(*_model_graph(X, 10, 3.0, "asym_order"), 200).toarray()
    assert not np.array_equal(S, S.T)


def _solve_case(seed=1, n=120, k=8, kq=4, alpha=0.95, tol=1e-10, iters=400):
    X = _data("clustered", n=n, dim=16, seed=seed)
    Q = _data("clustered", n=6, dim=16, seed=seed)
    S = M.to_csr(*_model_graph(X, k, 3.0), n)
    qi, qs = M.topk_lists(M.exact_scores(X, Q), kq)
    return S, M.seeds(qi, qs, n, 3.0), alpha, tol, iters


def test_cg_agrees_with_a_dense_solve_within_the_residual_bound():
    S, Y, alpha, tol, iters = _solve_case()
    f, it, res = M.solve(S, Y, alpha, iters, tol)
    n = S.shape[0]
    for q in range(Y.shape[1]):
        fs = M.dense_solve(S, Y[:, q], alpha)
        true = M.true_residual(S, Y[:, q], f[q], alpha)
        # ||f - f*|| <= ||y - (I - aS) f|| / (1 - a), plus the dense solve's own error (backward error n u ||A|| ||f*||)
        bound = (true + 2 * n * M.U * (1 + alpha) * np.linalg.norm(fs)) / (1 - alpha)
        assert np.linalg.norm(f[q] - fs) <= bound
        assert it[q] < iters and res[q] <= tol * np.linalg.norm(Y[:, q])


@pytest.mark.parametrize("bug", ["drop_row", "rr_tol"])
def test_planted_solver_bugs_leave_the_residual_check(bug):
    S, Y, alpha, _, iters = _solve_case()
    tol = 1e-4

    def worst(b):
        f, it, _ = M.solve(S, Y, alpha, iters, tol, b)
        return max(M.true_residual(S, Y[:, q], f[q], alpha) / (tol * np.linalg.norm(Y[:, q])) for q in range(Y.shape[1]))
    assert worst(None) <= 1 + 1e-6
    assert worst(bug) > 1.5


def test_zero_seed_gives_zero():
    S, Y, alpha, tol, iters = _solve_case()
    f, it, res = M.cg(S, np.zeros(S.shape[0]), alpha, iters, tol)
    assert not f.any() and it == 0 and res == 0


def test_rank_counts_follow_the_stable_argsort():
    f = np.array([0.5, 0.0, -0.0, 0.5, 1.0, 0.0, -1.0, 0.5])
    order = M.ranking(f)
    pos = np.empty_like(order)
    pos[order] = np.arange(f.size)
    rows = np.arange(f.size)
    assert np.array_equal(M.rank_counts(f, rows, np.ones(f.size, np.uint8)), pos)
    assert np.array_equal(order, [4, 0, 3, 7, 1, 2, 5, 6])          # -0 == +0, ties -> lower index


def test_planted_manifold_diffusion_beats_plain_ranking():
    X, Q, pos = M.planted_manifold()
    p = dict(k=5, kq=3, gamma=3.0, alpha=0.99, iters=50, tol=0.0)
    f, _, _, _ = M.diffuse(X, Q, **p)
    plain = np.mean([M.average_precision(M.ranking(M.exact_scores(X, Q)[q]), pos[q]) for q in range(len(pos))])
    diff = np.mean([M.average_precision(M.ranking(f[q]), pos[q]) for q in range(len(pos))])
    assert plain < 0.75 and diff > plain + 0.2, (plain, diff)


def test_parameter_validation():
    from dirb200.diffusion import Diffusion, check_params
    check_params(k=1, kq=1, gamma=0.5, alpha=0.0, iters=1, tol=0.0)
    for bad in (dict(k=0), dict(k=2.5), dict(kq=0), dict(gamma=0), dict(gamma=-1), dict(alpha=1.0), dict(alpha=-0.1),
                dict(iters=0), dict(tol=-1e-9)):
        with pytest.raises(ValueError):
            check_params(**bad)
    with pytest.raises(ValueError):                   # refused before any device work
        Diffusion(np.zeros((3, 4), np.float32), k=0)


def test_diffusion_argument_parsing():
    from dirb200.diffusion import DEFAULTS
    from dirb200.pipeline import diffusion_params
    assert diffusion_params([50, 10]) == DEFAULTS
    assert diffusion_params([7.0, 3.0, 2.0, 0.5]) == dict(DEFAULTS, k=7, kq=3, gamma=2.0, alpha=0.5)
    for bad in ([5], [5, 3, 2, 0.5, 1], [0, 3], [5.5, 3], [5, 3, -1], [5, 3, 3, 1.0]):
        with pytest.raises(ValueError):
            diffusion_params(bad)
    from dirtorch import test_dir
    with pytest.raises(SystemExit):
        test_dir.test_dir_main(["--dataset", "Oxford5K", "--checkpoint", "none", "--diffusion", "5"])


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "diffusion.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+diffusion_cu\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 20
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
