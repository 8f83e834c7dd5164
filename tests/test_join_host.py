"""CPU checks of the range search / self-join model (tests/join_model.py): the kernel's triangle schedule covers every
needed tile once, the model agrees with a dense restatement of rules J2-J4 and with scipy's connected components, each
planted bug leaves a check, the command line's parsing and errors, and the new kernels build without spills."""
import os
import re

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

import join_model as M
from conftest import REPO

EPS16 = 1e-3


def _data(n, dim=16, seed=0, dup=True):
    """Clustered unit rows, some repeated: -> (E exact fp64 scores, F fp32 scores within EPS16 of E)."""
    r = np.random.RandomState(seed)
    c = r.standard_normal((max(2, n // 20), dim))
    X = c[r.randint(0, c.shape[0], n)] + 0.25 * r.standard_normal((n, dim))
    if dup and n > 12:
        X[5:8] = X[0]
        X[n - 3:] = X[9:12]
    X = (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)
    E = X.astype(np.float64) @ X.astype(np.float64).T
    F = (E + r.uniform(-0.9, 0.9, E.shape) * EPS16).astype(np.float32)
    return E, F


def _dense_pairs(E, tau):
    """J3 restated densely: for each i the j > i with e >= tau, ordered (e desc, j asc)."""
    n = E.shape[0]
    off, cols, sc = [0], [], []
    for i in range(n):
        j = np.arange(i + 1, n)
        j = j[E[i, j] >= tau]
        o = np.lexsort((j, -E[i, j]))
        cols.append(j[o])
        sc.append(E[i, j[o]])
        off.append(off[-1] + len(j))
    return np.array(off), np.concatenate(cols + [np.zeros(0, np.int64)]), np.concatenate(sc + [np.zeros(0)])


def _same(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))


def _scipy_labels(off, cols, n):
    g = sp.csr_matrix((np.ones(len(cols)), cols, off), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    first = {}
    for i, l in enumerate(lab):                       # relabel each component by its smallest row
        first.setdefault(l, i)
    return np.array([first[l] for l in lab], np.int64)


# ------------------------------------------------------------------------------------------------ triangle schedule
def _global_tiles(N, row_block, bug=None):
    """Every (row tile, column tile) the self-join of N rows launches, with blocks of row_block rows."""
    out = []
    for i0 in range(0, N, row_block):
        M_ = min(row_block, N - i0)
        b = i0 // M.TILE
        out += [(b + m, b + n) for m, n in M.block_tiles(M_, N - i0, bug)]
    return out


@pytest.mark.parametrize("row_block", [128, 256, 384, None])
def test_schedule_launches_every_needed_tile_once(row_block):
    for N in range(1, 1001):
        T = -(-N // M.TILE)
        tiles = _global_tiles(N, row_block or N)
        want = {(a, b) for a in range(T) for b in range(a, T)}
        assert len(tiles) == len(set(tiles)) == len(want), N
        assert set(tiles) == want, N
    assert len(M.block_tiles(1000, 1000)) == 8 * 9 // 2


def test_schedule_decode_over_large_grids():
    """The closed-form decode (sqrt and its corrections) at column counts where fp64 rounding matters."""
    for mt in (1, 2, 3, 1000, 8000):
        for t in list(range(0, min(mt * (mt + 1) // 2, 5000))) + [mt * (mt + 1) // 2 - 1, mt * (mt + 1) // 2, mt * (mt + 1) // 2 + 7]:
            m, n = M.decode_tri(t, mt)
            if t < mt * (mt + 1) // 2:
                assert n * (n + 1) // 2 + m == t and 0 <= m <= n < mt
            else:
                assert n >= mt and 0 <= m < mt


def test_planted_schedule_bug_skips_the_diagonal():
    tiles = _global_tiles(300, 128, bug="off_diagonal")
    assert (0, 0) not in tiles
    E, F = _data(300)
    assert not _same(M.self_join(E, F, 0.9, EPS16, row_block=128, bug="off_diagonal"), _dense_pairs(E, 0.9))


# ------------------------------------------------------------------------------------------------ model vs dense
@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 300])
@pytest.mark.parametrize("tau", [0.95, 0.8, 0.0, -1.0, 2.0])
def test_self_join_matches_dense(n, tau):
    E, F = _data(n, seed=n)
    want = _dense_pairs(E, tau)
    for row_block, cap in ((None, None), (128, 1), (256, 7)):
        assert _same(M.self_join(E, F, tau, EPS16, row_block=row_block, cap=cap), want), (row_block, cap)
    # J3: the self-join is the range search of the rows against themselves without j <= i
    off, rows, sc = M.range_search(E, F, tau, EPS16)
    keep = rows > np.repeat(np.arange(n), np.diff(off))
    off2 = np.concatenate([[0], np.cumsum([keep[off[i]:off[i + 1]].sum() for i in range(n)])])
    assert _same((off2, rows[keep], sc[keep]), want)


def test_range_search_is_inclusive_and_ordered():
    E, F = _data(200, seed=4)
    tau = float(np.sort(E[3])[-10])                    # exactly a score of row 3: inclusive boundary
    off, rows, sc = M.range_search(E, F, tau, EPS16)
    got = rows[off[3]:off[3 + 1]]
    assert len(got) == int((E[3] >= tau).sum()) and E[3, got[-1]] == tau
    for q in range(200):
        r, s = rows[off[q]:off[q + 1]], sc[off[q]:off[q + 1]]
        assert np.all((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (r[:-1] < r[1:])))


@pytest.mark.parametrize("seed", range(4))
def test_groups_match_scipy(seed):
    E, F = _data(260, seed=seed)
    off, cols, _ = M.self_join(E, F, 0.9, EPS16, row_block=128)
    labels = M.components(off, cols, 260)
    assert np.array_equal(labels, _scipy_labels(off, cols, 260))
    g = M.groups(labels)
    assert [int(x[0]) for x in g] == sorted(int(x[0]) for x in g)
    assert all(np.all(np.diff(x) > 0) and len(x) >= 2 for x in g)
    assert sum(len(x) for x in g) == sum(int((labels == l).sum()) for l in np.unique(labels) if (labels == l).sum() >= 2)


def test_components_edge_cases():
    n = 10000                                           # a chain: one component, label 0 everywhere
    off = np.arange(n + 1).clip(max=n - 1)
    cols = np.arange(1, n)
    assert np.array_equal(M.components(off, cols, n), np.zeros(n, np.int64))
    assert np.array_equal(M.components(np.zeros(6, np.int64), np.zeros(0, np.int64), 5), np.arange(5))
    assert M.groups(np.arange(5)) == []


# ------------------------------------------------------------------------------------------------ planted bugs
def test_planted_diagonal_bug():
    E, F = _data(200)
    got = M.self_join(E, F, 0.9, EPS16, bug="keep_diagonal")
    assert not _same(got, _dense_pairs(E, 0.9))


def test_planted_rounding_bug():
    """J5 itself: thr <= tau - eps16 < the next fp32 above thr, over many (tau, eps16)."""
    r = np.random.RandomState(0)
    caught = 0
    for tau, eps in zip(r.uniform(-1, 1, 2000), r.uniform(1e-4, 5e-3, 2000)):
        x = float(tau) - float(eps)
        t = M.threshold(tau, eps)
        assert float(t) <= x < float(np.nextafter(t, np.float32(np.inf)))
        caught += float(M.threshold(tau, eps, bug="round_nearest")) > x
    assert caught > 500


def test_planted_truncation_bug():
    E, F = _data(300, seed=2)
    want = M.self_join(E, F, 0.5, EPS16)
    assert _same(M.self_join(E, F, 0.5, EPS16, row_block=128, cap=3), want)
    assert not _same(M.self_join(E, F, 0.5, EPS16, row_block=128, cap=3, bug="truncate"), want)


def test_planted_first_seen_labels():
    E, F = _data(260, seed=1)
    off, cols, _ = M.self_join(E, F, 0.9, EPS16)
    assert not np.array_equal(M.components(off, cols, 260, bug="first_seen"), _scipy_labels(off, cols, 260))


# ------------------------------------------------------------------------------------------------ command line
def test_cli_parsing_and_errors():
    from dirb200 import duplicates as D
    a = D.parse_args(["--load-feats", "x.npy", "--threshold", "0.9", "--output", "o.npz"])
    assert a.threshold == 0.9 and a.load_feats == "x.npy" and a.output == "o.npz" and a.gpu == 0
    a = D.parse_args(["--dataset", "ImageList('l.txt')", "--checkpoint", "c.pt", "--threshold", "0.8", "--whiten",
                      "W", "--whitenp", "0.25", "--trfs", "", "--out-json", "g.json"])
    assert a.whiten == "W" and a.whitenp == 0.25 and a.out_json == "g.json"
    a = D.parse_args(["--store", "S", "--threshold", "0.5", "--against", "b.npy", "--gpu", "1"])
    assert a.against == "b.npy" and a.gpu == 1
    for bad in (["--load-feats", "x.npy"],                                           # no threshold
                ["--threshold", "0.9"],                                              # no input
                ["--load-feats", "x.npy", "--store", "S", "--threshold", "0.9"],     # two inputs
                ["--load-feats", "x.npy", "--threshold", "inf"],
                ["--load-feats", "x.npy", "--threshold", "nan"],
                ["--dataset", "D", "--threshold", "0.9"],                           # no checkpoint
                ["--load-feats", "x.npy", "--threshold", "0.9", "--eps16", "-1"],
                ["--load-feats", "x.npy", "--threshold", "0.9", "--against", "b.npy", "--out-json", "g.json"]):
        with pytest.raises(SystemExit):
            D.parse_args(bad)
    for bad in (float("nan"), float("inf"), "x", None):
        with pytest.raises(ValueError):
            D.check_tau(bad)
        with pytest.raises(ValueError):
            D.near_duplicates(np.zeros((4, 64), np.float32), bad)


def test_dirtorch_exports():
    from dirtorch import duplicates, find_duplicates
    from dirb200 import duplicates as D
    assert duplicates.near_duplicates is D.near_duplicates and duplicates.overlap is D.overlap
    assert find_duplicates.find_duplicates_main is D.find_duplicates_main


# ------------------------------------------------------------------------------------------------ build
def _stats(log, pattern):
    text = open(log).read()
    return re.findall(r"Compiling entry function '(%s)'.*?\n.*?\n(.*?)\n" % pattern, text)


def test_new_kernels_do_not_spill():
    build = os.path.join(REPO, "deep-image-retrieval_b200", "build")
    if not os.path.exists(os.path.join(build, "join.cu.log")):
        pytest.skip("no compiler log: the library was not built in this tree")
    blocks = _stats(os.path.join(build, "join.cu.log"), r"\w+join_cu\w+")
    blocks += _stats(os.path.join(build, "search.cu.log"), r"\w+join_(?:rescore|kept|emit)_kernel\w+")
    blocks += _stats(os.path.join(build, "search.cu.log"), r"_ZN4dirb16conv_pers_kernelILi128ELi6ELi5E\w+")
    assert len(blocks) == 6 + 3 + 1
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
