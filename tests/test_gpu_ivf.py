"""Inverted-file search on the GPU (DESIGN.md section 4.10, rules I1-I7).  -m gpu

With every list probed the result must be Index.search bit for bit; with fewer it must equal tests/ivf_model.py and
the exact search of the probed rows alone, bit for bit, whatever the candidate capacity, workspace or run."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_model as M  # noqa: E402
import kmeans_model as KM  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mods():
    from dirb200 import ivf, ops
    ops.require_gpu(0)
    return ivf, ops


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _clustered(n, dim, k, seed=0, spread=0.35):
    r = np.random.RandomState(seed)
    c = _unit(r.standard_normal((k, dim)))
    return _unit(c[r.randint(0, k, n)] + spread * r.standard_normal((n, dim)) / np.sqrt(dim / 64))


def _same(a, b):
    for x, y in zip(a, b):
        x, y = x.cpu().numpy(), y.cpu().numpy() if isinstance(y, torch.Tensor) else y
        assert x.shape == y.shape
        assert np.array_equal(x.view(np.uint8), np.ascontiguousarray(y, x.dtype).view(np.uint8))


def _exact(ops, X, q, k):
    idx = ops.Index(_t(X))
    try:
        return idx.search(_t(q), k)
    finally:
        idx.close()


@pytest.mark.parametrize("N,D,K,ks", [(6000, 64, 1, (1, 100, 1024, 1025, 5000)),
                                      (20000, 2048, 7, (1, 100, 1024, 1025, 5000)),
                                      (200000, 64, 1024, (1, 100, 1024, 1025, 5000))])
def test_all_lists_equal_the_exact_search(N, D, K, ks):
    ivf, ops = _mods()
    X = _clustered(N, D, max(K, 16), seed=N)
    r = np.random.RandomState(1)
    C = X[r.choice(N, K, replace=False)]
    q = _clustered(37, D, max(K, 16), seed=N + 1)
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        for k in ks:
            _same(index.search(_t(q), k, K), _exact(ops, X, q, k))
    finally:
        index.close()


def _small_case(seed=3, N=3000, D=64, K=37):
    """Clustered rows; centre K-1 duplicates centre 0 (an empty list, probe ties) and centre K-2 is a lone row."""
    X = _clustered(N, D, K - 2, seed=seed, spread=0.05)
    r = np.random.RandomState(seed)
    C = np.concatenate([_unit(r.standard_normal((K - 2, D))), np.zeros((2, D), np.float32)])   # _clustered's centres
    X[-1] = _unit(r.standard_normal((1, D)))[0]
    C[K - 2] = X[-1]
    C[K - 1] = C[0]
    q = np.concatenate([_clustered(30, D, K - 2, seed=seed, spread=0.1)[::-1], C[:1]])
    return X, C, q


def test_partial_probes_equal_the_model():
    ivf, ops = _mods()
    X, C, q = _small_case()
    E = KM.exact_scores(q, X)
    Ec = KM.exact_scores(q, C)
    labels = KM.assign(KM.exact_scores(X, C))[0]
    perm, off = M.build(labels, C.shape[0])
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        assert np.array_equal(index.labels_.cpu().numpy(), labels)
        sizes = index.list_sizes_.cpu().numpy()
        assert sizes[-1] == 0 and sizes[-2] == 1
        for nprobe in (1, 3, 10, 36):
            probes = M.probe(Ec, nprobe)
            assert np.array_equal(index.probe(_t(q), nprobe).cpu().numpy(), probes)
            for k in (1, 50, 400, 3500):
                got = index.search(_t(q), k, nprobe)
                _same(got, M.search(E, probes, perm, off, k))
                # the exact search of the probed rows alone, its indices mapped back (rule I4)
                for i in (0, 7, q.shape[0] - 1):
                    R = np.sort(M.union(probes[i], perm, off))
                    s, ix = _exact(ops, X[R], q[i:i + 1], k)
                    ix = ix.cpu().numpy()
                    assert np.array_equal(got[1][i].cpu().numpy(), np.where(ix[0] >= 0, R[np.maximum(ix[0], 0)], -1))
                    assert np.array_equal(got[0][i].cpu().numpy().view(np.uint8), s[0].cpu().numpy().view(np.uint8))
    finally:
        index.close()


def test_more_than_65535_pairs_in_one_list():
    ivf, ops = _mods()
    X = _clustered(2000, 64, 8, seed=5)
    q = _clustered(70000, 64, 8, seed=6)
    index = ivf.IVFIndex(_t(X), _t(X[:1]))
    try:
        _same(index.search(_t(q), 10, 1), _exact(ops, X, q, 10))
        assert index.stats()["pairs"] == 70000
    finally:
        index.close()


def test_every_probed_row_is_a_candidate_with_a_wide_band():
    ivf, _ = _mods()
    X, C, q = _small_case(seed=8, N=800, K=9)
    E = KM.exact_scores(q, X)
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        index.set_option("eps16", 10.0)
        probes = index.probe(_t(q), 2).cpu().numpy()
        got = index.search(_t(q), 10, 2)
        perm, off = index.perm_.cpu().numpy(), index.cell_off_.cpu().numpy()
        st = index.stats()
        assert st["candidates"] == st["probed_rows"] == sum(M.union(p, perm, off).shape[0] for p in probes)
        _same(got, M.search(E, probes, perm, off, 10))
    finally:
        index.close()


def test_overflow_workspace_and_runs_give_the_same_bits():
    ivf, _ = _mods()
    X, C, q = _small_case(seed=11, N=20000, D=128, K=40)
    q = np.concatenate([q] * 20)
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        ref = index.search(_t(q), 100, 5)
        assert index.stats()["reruns"] == 0
        _same(index.search(_t(q), 100, 5), ref)
        index.set_option("cand_cap", 1)
        _same(index.search(_t(q), 100, 5), ref)
        assert index.stats()["reruns"] >= 1
        index.set_option("cand_cap", 0)
        index.set_option("ws_budget", 3e6)
        _same(index.search(_t(q), 100, 5), ref)
        index.set_option("ws_budget", 4.0 * (1 << 30))
        _same(index.search(_t(q), 1025, 5)[1][:, :100], ref[1])
    finally:
        index.close()


def test_rank_counts_follow_rule_i7():
    ivf, ops = _mods()
    X, C, q = _small_case(seed=13)
    E = KM.exact_scores(q, X)
    r = np.random.RandomState(0)
    t_off = np.arange(0, 6 * q.shape[0] + 1, 6, dtype=np.int32)
    t_rows = r.randint(0, X.shape[0], t_off[-1]).astype(np.int64)
    t_flags = np.ones(t_rows.shape[0], np.uint8)
    t_q = np.repeat(np.arange(q.shape[0]), 6)
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        _, a_all = index.index.rank_counts(_t(q), t_off, t_rows, t_flags)
        _, _, full = index.rank_counts(_t(q), t_off, t_rows, t_flags, C.shape[0])
        assert np.array_equal(full.cpu().numpy(), a_all.cpu().numpy())
        perm, off = index.perm_.cpu().numpy(), index.cell_off_.cpu().numpy()
        for nprobe in (1, 4):
            inside, _, got = index.rank_counts(_t(q), t_off, t_rows, t_flags, nprobe)
            probes = M.probe(KM.exact_scores(q, C), nprobe)
            want = M.ranks(E, probes, perm, off, t_q, t_rows)
            assert np.array_equal(got.cpu().numpy(), want)
            assert np.array_equal(inside.cpu().numpy(),
                                  [t in set(M.union(probes[a], perm, off)) for a, t in zip(t_q, t_rows)])
    finally:
        index.close()


def test_errors():
    ivf, _ = _mods()
    X, C, q = _small_case(seed=2, N=500, K=5)
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        for bad in (0, 6, 2.5):
            with pytest.raises(ValueError):
                index.search(_t(q), 5, bad)
        with pytest.raises(ValueError):
            index.search(_t(q), 0, 1)
        with pytest.raises(ValueError):
            index.search(_t(q[:, :32].copy()), 5, 1)
        with pytest.raises(ValueError):
            index.search(_t(2 * q), 5, 1)
    finally:
        index.close()
    with pytest.raises(ValueError):
        ivf.IVFIndex(_t(2 * X), _t(C))
    with pytest.raises(ValueError):
        ivf.IVFIndex(_t(X), _t(2 * C))
    with pytest.raises(ValueError):
        ivf.IVFIndex(_t(X), _t(C[:, :32].copy()))


def test_train_and_determinism():
    ivf, _ = _mods()
    X = _clustered(5000, 64, 20, seed=21)
    a = ivf.IVFIndex.train(_t(X), 16, seed=0, max_iter=5)
    b = ivf.IVFIndex(_t(X), a.kmeans_)
    try:
        assert torch.equal(a.perm_, b.perm_) and torch.equal(a.cell_off_, b.cell_off_)
        _same(a.search(_t(X[:50]), 20, 3), b.search(_t(X[:50]), 20, 3))
    finally:
        a.close()
        b.close()


def test_new_database_detaches_the_lists():
    ivf, ops = _mods()
    from dirb200 import lib
    X, C, q = _small_case(seed=4, N=500, K=5)
    index = ivf.IVFIndex(_t(X), _t(C))
    try:
        h = index.index
        lib.call("dirb200_index_set_db", h._h, ops._ptr(h.db32), ops._ptr(h.db16), h.n - 1, 0)
        with pytest.raises(lib.DirbError):
            h.search_lists(_t(q), 5, index.probe(_t(q), 2))
    finally:
        index.close()


def _band_lists(n):
    """Lists for the decoy / trap layout of tests/band_data.py: list 0 = the first rows (a decoy per group of 32, list
    size not a multiple of 128), list 1 = rows that are never probed, list 2 = the rest with every trap."""
    import band_data as B
    db, q, info = B.topk_layout(2048, n)
    labels = np.full(n, 2, np.int64)
    labels[:n // 2 + 37] = 0
    labels[n // 2 + 37:3 * n // 4] = 1
    labels[info["trap"]] = 2
    labels[info["decoy"]] = 0
    return db, q, info, labels


@pytest.mark.parametrize("probes", [[0, 2], [2, 0, 1]])
def test_band_edges_decoys_and_traps_through_the_lists(probes):
    """With k = the number of traps the exact top-k is the traps, while on the fp16 path every decoy outranks them by
    more than 1.25 eps16 (less than 2 eps16): the band of rule I5 keeps them.  With eps16 at 0.45 x the gap the H100
    produced, the list search must come out wrong - the test depends on the full band."""
    _, ops = _mods()
    import oracle.dir_oracle as O
    from test_gpu_band_edges import _gap
    db, q, info, labels = _band_lists(20000)
    k = info["k"]
    perm, off = M.build(labels, 3)
    rs, ri = O.topk(q[None], db, k)
    assert set(ri[0]) == set(info["trap"])
    index = ops.Index(_t(db), check_norms=False)
    try:
        index.set_lists(index.db16[_t(perm)].contiguous(), _t(perm), _t(off))
        pr = _t(np.array([probes], np.int64))
        s, i = index.search_lists(_t(q[None]), k, pr)
        assert np.array_equal(i.cpu().numpy(), ri) and np.array_equal(s.cpu().numpy(), rs)
        # the seed came from the decoys (one per group of 32 rows of list 0), so the traps were candidates only by the band
        assert index.lists_stats()["candidates"] >= len(info["decoy"]) + k
        gap = _gap(ops, q, db, info["decoy"], info["trap"])
        index.set_option("eps16", 0.45 * gap)
        s, i = index.search_lists(_t(q[None]), k, pr)
        assert not np.array_equal(i.cpu().numpy(), ri) and not set(i.cpu().numpy()[0]) & set(info["trap"])
    finally:
        index.close()


def _oxford_aps_i7(E, probes, perm, off, gnd):
    """Rule I7's list L_q, junk removed, AP of the positives (the numpy model end to end)."""
    from dirb200.datasets import compute_average_precision
    aps = []
    for qi, g in enumerate(gnd):
        R = set(M.union(probes[qi], perm, off).tolist())
        key = lambda r: (r not in R, -E[qi, r], r)
        junk = set(g["junk"])
        order = [r for r in sorted(range(E.shape[1]), key=key) if r not in junk]
        rank = {r: i for i, r in enumerate(order)}
        aps.append(compute_average_precision(np.sort([rank[p] for p in g["ok"]])))
    return aps


def test_dir_main_with_ivf(tmp_path, monkeypatch):
    """test_dir --ivf on the synthetic Oxford layout: every list probed gives the APs of the default rank-count path
    exactly; fewer lists give the APs of the numpy model of rule I7; with --aqe (queries probed after the expansion)
    and --whiten (lists built on the whitened rows)."""
    _mods()
    import e2e_data
    from sklearn.decomposition import PCA
    from dirb200.ivf import IVFIndex
    from dirb200.pipeline import expand_descriptors
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root, hard=True)
    ckpt = os.path.join(root, "ckpt.pt")
    opts = dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_options": opts}, ckpt)
    monkeypatch.setenv("DB_ROOT", root)
    from dirtorch import test_dir
    saved = os.path.join(root, "saved")
    base = ["--dataset", "Oxford5K", "--checkpoint", ckpt, "--whiten", "", "--gpu", "0", "--threads", "2", "--detailed"]
    res = test_dir.test_dir_main(base + ["--ivf", "4", "1", "--save-feats", saved])
    B = np.load(os.path.join(saved, "feats.bdescs.npy"))
    qpath = os.path.join(saved, "feats.qdescs.npy")
    Qd = np.load(qpath) if os.path.exists(qpath) else B[qn]
    load = base + ["--load-feats", saved]
    for extra in ([], ["--aqe", "2", "1"]):
        plain = test_dir.test_dir_main(load + extra)
        full = test_dir.test_dir_main(load + extra + ["--ivf", "4", "4"])
        assert full["APs"] == plain["APs"]
    lists = IVFIndex.train(_t(B), 4, seed=0)
    C = lists.kmeans_.cluster_centers_.cpu().numpy()
    lists.close()
    labels = KM.assign(KM.exact_scores(B, C))[0]
    perm, off = M.build(labels, 4)
    Qa = expand_descriptors(_t(Qd), db=_t(B), k=2, alpha=1.0)
    for extra, q, nprobe in (([], Qd, 1), (["--aqe", "2", "1"], np.asarray(Qa, np.float32), 1), ([], Qd, 2)):
        r = test_dir.test_dir_main(load + extra + ["--ivf", "4", str(nprobe)])
        want = _oxford_aps_i7(KM.exact_scores(q, B), M.probe(KM.exact_scores(q, C), nprobe), perm, off, gnd)
        np.testing.assert_allclose(r["APs"], want, rtol=0, atol=1e-12)
    assert res["APs"] == test_dir.test_dir_main(load + ["--ivf", "4", "1"])["APs"]
    # whitening: the lists are built on the whitened rows; every list probed is again the default path
    pca = PCA(n_components=32, whiten=True).fit(B)
    ckpt_w = os.path.join(root, "ckpt_w.pt")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_options": opts, "pca": {"W": pca}}, ckpt_w)
    wl = ["--dataset", "Oxford5K", "--checkpoint", ckpt_w, "--whiten", "W", "--gpu", "0", "--load-feats", saved, "--detailed"]
    assert test_dir.test_dir_main(wl + ["--ivf", "4", "4"])["APs"] == test_dir.test_dir_main(wl)["APs"]
    aps = test_dir.test_dir_main(wl + ["--ivf", "4", "1"])["APs"]
    assert len(aps) == len(gnd) and all(0 <= a <= 1 for a in aps)
