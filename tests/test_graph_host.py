"""Graph search on the CPU (DESIGN.md section 4.12): the model of tests/graph_model.py against plain-loop restatements
of rules G3-G5 and G7's identity, five planted bugs, the --graph parsing, the shared-memory limit and spills."""
import os
import re

import numpy as np
import pytest

import graph_model as GM
import kmeans_model as KM
from conftest import REPO


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _knn_exact(X, K):
    E = KM.exact_scores(X, X)
    return np.lexsort((np.broadcast_to(np.arange(X.shape[0]), E.shape), -E), axis=1)[:, :K + 1]


def _detours_loop(knn):
    n, K = knn.shape
    out = np.zeros((n, K), np.int64)
    for r in range(n):
        for j in range(K):
            nj = knn[r, j]
            if nj < 0:
                continue
            for i in range(j):
                ni = knn[r, i]
                if ni >= 0 and any(knn[ni, p] == nj for p in range(j)):
                    out[r, j] += 1
    return out


def _graph_loop(knn, degree):
    n, K = knn.shape
    det = _detours_loop(knn)
    F = []
    for r in range(n):
        cand = sorted([(det[r, j], j) for j in range(K) if knn[r, j] >= 0])[:degree]
        F.append([int(knn[r, j]) for _, j in cand])
    rev = [[] for _ in range(n)]
    for pos in range(degree):
        for s in range(n):
            if pos < len(F[s]):
                rev[F[s][pos]].append(s)
    G = np.full((n, degree), -1, np.int64)
    for r in range(n):
        g = F[r][:degree // 2]
        for c in rev[r] + F[r][degree // 2:]:
            if len(g) < degree and c not in g:
                g.append(c)
        G[r, :len(g)] = g
    return G


def _cases():
    r = np.random.RandomState(0)
    X = _unit(r.standard_normal((60, 16)))
    X[7] = X[3]                                   # duplicates: row 7 may drop out of its own list
    X[9] = X[3]
    Xt = _unit(np.repeat(r.standard_normal((6, 16)), 10, axis=0) + 1e-3 * r.standard_normal((60, 16)))   # tie-heavy
    out = []
    for Y, K in ((X, 12), (Xt, 15), (X[:1], 0), (X[:2], 1), (X[:5], 4)):
        out.append(GM.knn_lists(_knn_exact(Y, K), K))
    holes = out[0].copy()
    holes[r.rand(*holes.shape) < 0.2] = -1            # -1 padding
    out.append(holes)
    return out


@pytest.mark.parametrize("case", range(6))
@pytest.mark.parametrize("degree", [1, 4, 7, 30])
def test_build_equals_loops(case, degree):
    knn = _cases()[case]
    assert np.array_equal(GM.detours(knn), _detours_loop(knn))
    F = GM.forward(knn, degree)
    assert np.array_equal(GM.merge(F, GM.reverse(F), degree), _graph_loop(knn, degree))


def test_self_removal():
    idx = np.array([[0, 1, 2], [0, 1, 2], [0, 1, 3], [1, 3, -1]])
    assert GM.knn_lists(idx, 2).tolist() == [[1, 2], [0, 2], [0, 1], [1, -1]]


def test_every_row_visited_is_dense_top_k():
    r = np.random.RandomState(1)
    X = _unit(r.standard_normal((120, 32)))
    q = _unit(r.standard_normal((4, 32)))
    G = GM.build(_knn_exact(X, 20), 20, 16)
    E = KM.exact_scores(q, X)
    Ent = GM.entry(120, 30, 0)
    for i in range(4):
        sc, ix, V, it = GM.search(E[i], G, GM.seeds(E[i], Ent, 4), 10, 120, 2, 500)
        assert sorted(V) == list(range(120))
        order = np.lexsort((np.arange(120), -E[i]))[:10]
        assert ix.tolist() == order.tolist() and np.array_equal(sc, E[i, order])
        assert np.array_equal(GM.ranks(E[i], V, np.arange(120)), np.argsort(order.tolist() + [
            j for j in np.lexsort((np.arange(120), -E[i])) if j not in set(order.tolist())]))


def test_planted_bugs_are_caught():
    r = np.random.RandomState(2)
    X = _unit(r.standard_normal((300, 16)))
    q = _unit(r.standard_normal((6, 16)))
    idx = _knn_exact(X, 16)
    caught = set()
    ref = GM.build(idx, 16, 8)
    for bug in ("detour_le", "rev_reversed"):
        if not np.array_equal(GM.build(idx, 16, 8, bug), ref):
            caught.add(bug)
    E = KM.exact_scores(q, X)
    E[:, 41] = E[:, 40]                                  # a planted score tie
    Ent = GM.entry(300, 64, 0)
    for bug in ("parents_ignore_flag", "row_desc", "dedupe_against_b"):
        for i in range(6):
            e = E[i].copy()
            sd = GM.seeds(e, Ent, 4)
            if bug == "row_desc":
                e[sd[0]] = e[sd[1]]                      # a tie inside B
            a = GM.search(e, ref, sd, 8, 8, 1, 30)
            b = GM.search(e, ref, sd, 8, 8, 1, 30, bug)
            if a[1].tolist() != b[1].tolist() or a[2] != b[2] or a[3] != b[3]:
                caught.add(bug)
    assert caught == {"detour_le", "rev_reversed", "parents_ignore_flag", "row_desc", "dedupe_against_b"}


def test_graph_argument_parsing():
    from dirb200.pipeline import graph_params
    assert graph_params([32, 128]) == dict(degree=32, itopk=128)
    for bad in ([32], [32, 128, 1], [0, 10], [32, 0], [1.5, 10], [129, 10]):
        with pytest.raises(ValueError):
            graph_params(bad)
    from dirtorch import test_dir
    for argv in (["--graph", "8", "16", "--ivf", "4", "2"], ["--graph", "8", "16", "--diffusion", "5", "3"],
                 ["--graph", "8"], ["--graph", "8", "0"]):
        with pytest.raises(SystemExit):
            test_dir.test_dir_main(["--dataset", "Oxford5K", "--checkpoint", "none"] + argv)


def test_shared_memory_limit():
    from dirb200 import graph
    table = [(16, 128, 1, 32, 256, 137416), (16, 128, 1, 32, 0, 6472), (1, 1, 1, 1, 0, 168),
             (64, 512, 4, 64, 100, 291920), (16, 128, 1, 32, 512, 268488)]
    assert [(*row[:5], graph.smem_bytes(*row[:5])) for row in table] == table
    assert graph.smem_bytes(0, 128, 1, 32, 10) == 0 and graph.smem_bytes(16, 128, 1, 32, -1) == 0
    h100 = 232448                                        # 227 KB, the H100's per-block opt-in limit
    assert graph.max_iter_limit(h100, 16, 128, 1, 32) == 511
    assert graph.max_iter_limit(h100, 16, 128, 4, 64) == 63
    assert graph.max_iter_limit(1000, 16, 128, 1, 32) == -1
    for args in ((16, 128, 1, 32), (8, 32, 1, 16), (100, 1000, 2, 50)):
        m = graph.max_iter_limit(h100, *args)
        assert graph.smem_bytes(*args, m) <= h100 < graph.smem_bytes(*args, m + 1)


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "graph.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+graph_\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 3
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
