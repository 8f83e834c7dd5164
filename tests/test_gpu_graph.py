"""Graph search on the GPU (DESIGN.md section 4.12, rules G1-G8).  -m gpu

graph_ must equal tests/graph_model.py bit for bit; results, fp64 score bits, visited lists in arrival order, |V| and
iteration counts must equal the model; the result must be the exact search of the visited rows, and with every row
visited Index.search itself."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import graph_model as GM  # noqa: E402
import kmeans_model as KM  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mods():
    from dirb200 import graph, lib, ops
    ops.require_gpu(0)
    return graph, ops, lib


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _data(n, d, nq, seed=0, clusters=None):
    r = np.random.RandomState(seed)
    if clusters:
        C = r.standard_normal((clusters, d))
        X = _unit(C[r.randint(0, clusters, n)] + 0.3 * r.standard_normal((n, d)))
    else:
        X = _unit(r.standard_normal((n, d)) * np.exp(-np.arange(d) / (d / 4)))
    if n > 12:
        X[11] = X[5]                                          # exact duplicates: equal scores, ties to the smaller row
        X[12] = X[5]
    q = _unit(X[r.randint(0, n, nq)] + 0.2 * r.standard_normal((nq, d)) / np.sqrt(d / 16))
    return X, q


def _knn_idx(ops, X, K):
    index = ops.Index(_t(X))
    try:
        return index.search(_t(X), K + 1)[1].cpu().numpy()
    finally:
        index.close()


@pytest.mark.parametrize("n,d,build_k,degree", [(1, 64, 64, 32), (2, 64, 64, 32), (3, 64, 64, 8), (40, 64, 64, 32),
                                                (700, 64, 16, 5), (3000, 64, 64, 32), (2500, 2048, 32, 16),
                                                (1000, 64, 128, 128), (20000, 64, 32, 16)])
def test_build_equals_model(n, d, build_k, degree):
    graph, ops, _ = _mods()
    X, _ = _data(n, d, 1, seed=n)
    g = graph.GraphIndex(_t(X), degree=degree, build_k=build_k)
    try:
        K = min(build_k, n - 1)
        idx = _knn_idx(ops, X, K)
        want = GM.build(idx, K, degree)
        assert g.graph_.shape == (n, degree) and g.graph_.dtype == torch.int32
        assert np.array_equal(g.graph_.cpu().numpy(), want)
        if n <= 3000 and d == 64:                             # rule G2's lists are the exact ones
            E = KM.exact_scores(X, X)
            order = np.lexsort((np.broadcast_to(np.arange(n), E.shape), -E), axis=1)[:, :K + 1]
            assert np.array_equal(idx, order)
    finally:
        g.close()


def test_build_from_supplied_knn():
    graph, ops, _ = _mods()
    X, _ = _data(1500, 64, 1, seed=7)
    K, degree = 24, 12
    idx = _knn_idx(ops, X, K + 5)                             # wider than needed: the first K + 1 columns count
    sc = np.zeros(idx.shape)
    own = graph.GraphIndex(_t(X), degree=degree, build_k=K)
    sup = graph.GraphIndex(_t(X), degree=degree, build_k=K, knn=(sc, idx))
    try:
        assert torch.equal(own.graph_, sup.graph_)
    finally:
        own.close()
        sup.close()
    holes = idx.copy()
    r = np.random.RandomState(1)
    for row in r.choice(1500, 300, replace=False):            # -1 entries, also rows that lose themselves
        holes[row, r.randint(0, K + 1):K + 1] = -1
    holes[3, :K + 1] = np.roll(holes[3, :K + 1], 1)
    g = graph.GraphIndex(_t(X), degree=degree, build_k=K, knn=(sc, holes))
    try:
        assert np.array_equal(g.graph_.cpu().numpy(), GM.build(holes, K, degree))
    finally:
        g.close()


@pytest.fixture(scope="module")
def built():
    graph, _, _ = _mods()
    X, q = _data(3000, 64, 5000, seed=1)
    g = graph.GraphIndex(_t(X), degree=16, build_k=32, n_entry=64, seed=2)
    yield dict(g=g, X=X, q=q, G=g.graph_.cpu().numpy(), E=g.entry_.cpu().numpy())
    g.close()


def _check_against_model(b, qsel, k, itopk, width, max_iter, n_seeds, Q=None):
    g = b["g"]
    q = b["q"][:Q] if Q else b["q"][qsel]
    sc, ix = g.search(_t(q), k, itopk=itopk, width=width, max_iter=max_iter, n_seeds=n_seeds)
    st = g.stats()
    vs, vi = g.visited(_t(q), itopk=itopk, width=width, max_iter=max_iter, n_seeds=n_seeds)
    assert torch.equal(g.stats()["visited"], st["visited"]) and torch.equal(g.stats()["iterations"], st["iterations"])
    sc, ix, vs, vi = (t.cpu().numpy() for t in (sc, ix, vs, vi))
    nv, nit = st["visited"].cpu().numpy(), st["iterations"].cpu().numpy()
    rows = range(q.shape[0]) if not Q else qsel
    e_all = KM.exact_scores(b["q"][qsel] if Q else q, b["X"])
    for j, i in enumerate(rows):
        e = e_all[j]
        sd = GM.seeds(e, b["E"], n_seeds)
        ms, mi, V, it = GM.search(e, b["G"], sd, k, itopk, width, max_iter)
        assert ix[i].tolist() == mi.tolist(), i
        assert np.array_equal(sc[i].view(np.int64), ms.view(np.int64)), i
        assert nv[i] == len(V) and nit[i] == it, (i, nv[i], len(V), nit[i], it)
        assert vi[i, :len(V)].tolist() == V and (vi[i, len(V):] == -1).all()
        assert np.array_equal(vs[i, :len(V)].view(np.int64), e[V].view(np.int64))
    return sc, ix, vs, vi, nv


@pytest.mark.parametrize("k,itopk,width,max_iter,n_seeds", [
    (16, 16, 1, 64, 8),          # k = itopk
    (10, 32, 1, 256, 16),
    (4, 4, 8, 40, 4),            # width > the unexpanded entries of B
    (3, 64, 4, 30, 16),
    (7, 64, 1, 0, 16),           # seeds only
    (20, 40, 2, 50, 64),         # n_seeds = |E|
])
def test_search_equals_model(built, k, itopk, width, max_iter, n_seeds):
    _check_against_model(built, list(range(0, 60, 3)), k, itopk, width, max_iter, n_seeds)


def test_search_q1_q5000_and_largest_max_iter(built):
    graph, _, _ = _mods()
    g = built["g"]
    _check_against_model(built, [0], 10, 48, 1, 300, 16)
    sc, ix, _, _, nv = _check_against_model(built, list(range(0, 5000, 125)) + [4999], 10, 48, 1, 300, 16, Q=5000)
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    top = graph.max_iter_limit(limit, 8, 32, 1, 16)
    assert top > 1000
    assert graph.smem_bytes(8, 32, 1, 16, top) <= limit < graph.smem_bytes(8, 32, 1, 16, top + 1)
    _check_against_model(built, [1, 2, 3], 5, 32, 1, top, 8)
    with pytest.raises(ValueError, match="shared memory"):
        g.search(_t(built["q"][:2]), 5, itopk=32, width=1, max_iter=top + 1, n_seeds=8)


def test_result_is_exact_search_of_visited(built):
    _, ops, _ = _mods()
    g, X = built["g"], built["X"]
    q = built["q"][:12]
    sc, ix = g.search(_t(q), 25, itopk=64, width=2, max_iter=60, n_seeds=16)
    vs, vi = g.visited(_t(q), itopk=64, width=2, max_iter=60, n_seeds=16)
    for i in range(q.shape[0]):
        V = vi[i][vi[i] >= 0]
        sub = ops.Index(_t(X)[V].contiguous())
        s2, i2 = sub.search(_t(q[i:i + 1]), 25)
        sub.close()
        assert torch.equal(ix[i], V[i2[0]]) and torch.equal(sc[i].view(torch.int64), s2[0].view(torch.int64))


@pytest.mark.parametrize("k", [1, 100, 512])
def test_every_row_visited_is_index_search(k):
    graph, ops, _ = _mods()
    X, q = _data(500, 64, 30, seed=4)
    g = graph.GraphIndex(_t(X), degree=32, build_k=48, n_entry=100)
    exact = ops.Index(_t(X))
    try:
        assert g.n_components_ == 1
        sc, ix = g.search(_t(q), k, itopk=512, width=4, max_iter=100, n_seeds=8)
        assert (g.stats()["visited"] == 500).all()
        es, ei = exact.search(_t(q), k)
        assert torch.equal(ix, ei) and torch.equal(sc.view(torch.int64), es.view(torch.int64))
    finally:
        g.close()
        exact.close()


def test_dimension_not_a_multiple_of_64():
    """D = 100: the index pads rows and queries to 128 zero columns; search, visited and rank_counts take the caller's
    100-column queries and equal the model on the padded rows."""
    graph, _, _ = _mods()
    X, q = _data(1200, 100, 6, seed=9)
    Xp, qp = np.pad(X, ((0, 0), (0, 28))), np.pad(q, ((0, 0), (0, 28)))
    g = graph.GraphIndex(_t(X), degree=12, build_k=24, n_entry=200, device="cuda:0")
    try:
        assert g.x.shape == (1200, 128)
        from dirb200 import ops
        idx = _knn_idx(ops, Xp, 24)
        G = GM.build(idx, 24, 12)
        assert np.array_equal(g.graph_.cpu().numpy(), G)
        sc, ix = g.search(_t(q), 10, itopk=32, max_iter=50, n_seeds=8)
        vs, vi = g.visited(_t(q), itopk=32, max_iter=50, n_seeds=8)
        E = KM.exact_scores(qp, Xp)
        t_rows = np.random.RandomState(0).randint(0, 1200, 24)
        t_off = np.arange(0, 25, 4)
        inside, tsc, rank = g.rank_counts(_t(q), t_off, t_rows, np.ones(24, np.uint8), itopk=32, max_iter=50, n_seeds=8)
        Ent = g.entry_.cpu().numpy()
        for i in range(6):
            ms, mi, V, it = GM.search(E[i], G, GM.seeds(E[i], Ent, 8), 10, 32, 1, 50)
            assert ix[i].cpu().tolist() == mi.tolist()
            assert np.array_equal(sc[i].cpu().numpy().view(np.int64), ms.view(np.int64))
            assert vi[i, :len(V)].cpu().tolist() == V and (vi[i, len(V):] == -1).all()
            ts = t_rows[t_off[i]:t_off[i + 1]]
            assert np.array_equal(rank[t_off[i]:t_off[i + 1]].cpu().numpy(), GM.ranks(E[i], V, ts))
            assert inside[t_off[i]:t_off[i + 1]].cpu().tolist() == [t in set(V) for t in ts]
        with pytest.raises(ValueError):
            g.search(_t(qp), 10)                          # the padded width is not the index's dimension
    finally:
        g.close()


def test_determinism_reuse_and_components():
    graph, ops, _ = _mods()
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components
    X, q = _data(4000, 64, 200, seed=5, clusters=40)
    g = graph.GraphIndex(_t(X), degree=8, build_k=16, n_entry=256)
    try:
        a = g.search(_t(q), 10, itopk=32, max_iter=100)
        va = g.visited(_t(q), itopk=32, max_iter=100)
        b = g.search(_t(q), 10, itopk=32, max_iter=100)
        vb = g.visited(_t(q), itopk=32, max_iter=100)
        assert all(torch.equal(x.view(torch.int64) if x.is_floating_point() else x,
                               y.view(torch.int64) if y.is_floating_point() else y) for x, y in zip(a + va, b + vb))
        G = g.graph_.cpu().numpy()
        r, c = np.nonzero(G >= 0)
        want = connected_components(csr_matrix((np.ones(r.shape[0]), (r, G[r, c])), shape=(4000, 4000)),
                                    directed=True, connection="weak")[0]
        assert g.n_components_ == want and want > 1          # 40 tight clusters at degree 8 fall apart
        saved = graph.GraphIndex(_t(X), degree=8, build_k=16, n_entry=256, graph=g.graph_.cpu().numpy())
        idx = _knn_idx(ops, X, 16)
        sup = graph.GraphIndex(_t(X), degree=8, build_k=16, n_entry=256, knn=(None, idx))
        try:
            for h in (saved, sup):
                assert torch.equal(h.graph_, g.graph_) and h.n_components_ == g.n_components_
                s, i = h.search(_t(q), 10, itopk=32, max_iter=100)
                assert torch.equal(i, a[1]) and torch.equal(s.view(torch.int64), a[0].view(torch.int64))
        finally:
            saved.close()
            sup.close()
    finally:
        g.close()


def test_rank_counts_equal_model(built):
    g, X = built["g"], built["X"]
    q = built["q"][:8]
    r = np.random.RandomState(3)
    t_rows = r.randint(0, X.shape[0], 48)
    t_rows[:8] = g.visited(_t(q), itopk=32, max_iter=40)[1][:, 2].cpu().numpy()     # some targets inside V
    t_off = np.arange(0, 49, 6)
    flags = np.ones(48, np.uint8)
    flags[5] = 0
    inside, sc, rank = g.rank_counts(_t(q), t_off, t_rows, flags, itopk=32, max_iter=40)
    _, vi = g.visited(_t(q), itopk=32, max_iter=40)
    E = KM.exact_scores(q, X)
    for i in range(8):
        V = [v for v in vi[i].tolist() if v >= 0]
        ts = t_rows[t_off[i]:t_off[i + 1]]
        want = GM.ranks(E[i], V, ts)
        got = rank[t_off[i]:t_off[i + 1]].cpu().numpy()
        fl = flags[t_off[i]:t_off[i + 1]]
        assert np.array_equal(got, np.where(fl != 0, want, 0))
        assert inside[t_off[i]:t_off[i + 1]].cpu().numpy().tolist() == [t in set(V) for t in ts]
        assert np.array_equal(sc[t_off[i]:t_off[i + 1]].cpu().numpy().view(np.int64), E[i, ts].view(np.int64))


def test_errors(built):
    graph, _, _ = _mods()
    g = built["g"]
    q = _t(built["q"][:2])
    with pytest.raises(ValueError):
        g.search(q, 20, itopk=16)                             # k > itopk
    with pytest.raises(ValueError, match="shared memory"):
        g.search(q, 5, itopk=4096, width=8, max_iter=4096)
    with pytest.raises(ValueError):
        g.search(q, 5, n_seeds=65)                            # more seeds than the sample
    with pytest.raises(ValueError):
        g.search(_t(built["q"][:2, :32].copy()), 5)           # dimension mismatch
    with pytest.raises(ValueError):
        g.search(2 * q, 5)                                    # non-unit queries
    X = built["X"]
    with pytest.raises(ValueError):
        graph.GraphIndex(_t(2 * X[:100]))                     # non-unit rows
    for bad in (built["G"][:100], built["G"][:, :8], np.full((3000, 16), 3000), np.full((3000, 16), -2),
                built["G"].astype(np.float32)):
        with pytest.raises(ValueError):
            graph.GraphIndex(_t(X), degree=16, graph=bad)
    with pytest.raises(ValueError):
        graph.GraphIndex(_t(X), degree=129)


def _g8_aps(qd, bd, gnd, degree, itopk):
    """Rule G8's list from the numpy model on the descriptors the grading received, junk removed, AP of the
    positives (the graph is GraphIndex's on those rows, deterministic: the same as the grading's)."""
    from dirb200.datasets import compute_average_precision
    from dirb200.graph import GraphIndex
    g = GraphIndex(_t(bd), degree=degree)
    G, E0 = g.graph_.cpu().numpy(), g.entry_.cpu().numpy()
    g.close()
    n = bd.shape[0]
    E = KM.exact_scores(qd, bd)
    aps = []
    for qi, gq in enumerate(gnd):
        V = GM.traverse(E[qi], G, GM.seeds(E[qi], E0, 16), itopk, 1, 256)[0]
        inV, junk = set(V), set(gq["junk"])
        order = [r for r in sorted(range(n), key=lambda r: (r not in inV, -E[qi, r], r)) if r not in junk]
        rank = {r: i for i, r in enumerate(order)}
        aps.append(compute_average_precision(np.sort([rank[p] for p in gq["ok"]])))
    return aps, len(inV)


def test_dir_main_with_graph(tmp_path, monkeypatch):
    """test_dir --graph on the synthetic Oxford layout: a complete graph visits every row and gives the APs of the
    default rank-count path exactly; a sparse one gives the APs of the numpy model of rule G8 on the descriptors the
    grading receives; both with and without --aqe / --whiten."""
    _mods()
    import e2e_data
    from sklearn.decomposition import PCA
    from dirb200 import pipeline
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root, hard=True)
    ckpt = os.path.join(root, "ckpt.pt")
    opts = dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_options": opts}, ckpt)
    monkeypatch.setenv("DB_ROOT", root)
    from dirtorch import test_dir
    saved = os.path.join(root, "saved")
    base = ["--dataset", "Oxford5K", "--checkpoint", ckpt, "--whiten", "", "--gpu", "0", "--threads", "2", "--detailed"]
    test_dir.test_dir_main(base + ["--save-feats", saved])
    B = np.load(os.path.join(saved, "feats.bdescs.npy"))
    n = B.shape[0]
    load = base + ["--load-feats", saved]
    pca = PCA(n_components=32, whiten=True).fit(B)
    ckpt_w = os.path.join(root, "ckpt_w.pt")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_options": opts, "pca": {"W": pca}}, ckpt_w)
    wl = ["--dataset", "Oxford5K", "--checkpoint", ckpt_w, "--whiten", "W", "--gpu", "0", "--load-feats", saved, "--detailed"]
    seen = []
    orig = pipeline._aps_from_graph

    def record(db, qdescs, bdescs, params):
        seen.append((qdescs.cpu().numpy(), bdescs.cpu().numpy()))
        return orig(db, qdescs, bdescs, params)

    monkeypatch.setattr(pipeline, "_aps_from_graph", record)
    for argv in (load, load + ["--aqe", "2", "1"], wl, wl + ["--aqe", "2", "1"]):
        plain = test_dir.test_dir_main(argv)
        full = test_dir.test_dir_main(argv + ["--graph", str(n - 1), str(n)])
        assert full["APs"] == plain["APs"]
        seen.clear()
        r = test_dir.test_dir_main(argv + ["--graph", "2", "3"])
        (qd, bd), = seen
        want, last_v = _g8_aps(qd, bd, gnd, 2, 3)
        assert last_v < n
        np.testing.assert_allclose(r["APs"], want, rtol=0, atol=1e-12)
