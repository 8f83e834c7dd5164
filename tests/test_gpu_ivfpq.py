"""IVF-PQ on the GPU (DESIGN.md section 4.11, rules P1-P8).  -m gpu

Codebooks, codes, tables, candidates and results must equal tests/ivfpq_model.py bit for bit; with R at least the
probed rows the search must be IVFIndex.search bit for bit, and with every list probed and R >= N Index.search."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_model as IM  # noqa: E402
import ivfpq_model as P  # noqa: E402
import kmeans_model as KM  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mods():
    from dirb200 import ivf, ivfpq, lib, ops
    ops.require_gpu(0)
    return ivfpq, ivf, ops, lib


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _data(n, d, K, nq, seed=0):
    r = np.random.RandomState(seed)
    C = _unit(r.standard_normal((K, d)))
    X = _unit(C[r.randint(0, K, n)] + 0.5 * r.standard_normal((n, d)) / np.sqrt(d / 8))
    X[11] = X[5]                                            # equal rows: equal codes, ties to the smaller row
    q = _unit(X[r.randint(0, n, nq)] + 0.3 * r.standard_normal((nq, d)) / np.sqrt(d / 8))
    return X, C, q


def _model_lists(X, C):
    labels = KM.assign(KM.exact_scores(X, C))[0]
    perm, off = IM.build(labels, C.shape[0])
    return labels, perm, off


@pytest.mark.parametrize("d,M,n", [(64, 8, 3000), (64, 64, 3000), (2048, 32, 4000), (2048, 128, 4000),
                                   (2048, 8, 1500), (768, 8, 2000), (1280, 8, 1500)])
def test_build_equals_model(d, M, n):
    ivfpq, _, _, _ = _mods()
    X, C, q = _data(n, d, 5, 6)
    index = ivfpq.IVFPQIndex(_t(X), _t(C), M, train_size=600, pq_iter=2, seed=3)
    try:
        labels, perm, off = _model_lists(X, C)
        assert np.array_equal(index.perm_.cpu().numpy(), perm)
        CBs, empty = P.train(X, C, labels, M, 600, 2, 3)
        assert np.array_equal(index.codebooks_.cpu().numpy(), CBs)
        assert index.empty_codewords_ == empty
        sel = np.arange(0, n, max(1, n // 500))
        want = P.encode(P.residuals(X[perm[sel]], C, labels[perm[sel]]), CBs)
        assert np.array_equal(index.codes_.cpu().numpy()[sel], want)
        from dirb200 import lib, ops
        T = torch.empty((q.shape[0], M, 256), dtype=torch.float32, device=DEV)
        qt = _t(q)                                          # held: a temporary's block could be handed out again
        lib.call("dirb200_pq_tables", ops._ptr(qt), q.shape[0], d, ops._ptr(index.codebooks_), M, ops._ptr(T),
                 ops._stream())
        assert np.array_equal(T.cpu().numpy(), P.tables(q, CBs))
    finally:
        index.close()


def test_assign_ties_and_update_empty_codeword():
    _, _, ops, lib = _mods()
    r = np.random.RandomState(2)
    n, d, M = 600, 64, 8
    C = np.zeros((1, d), np.float32)
    CBs = r.standard_normal((M, 256, 8)).astype(np.float32)
    CBs[:, 11] = CBs[:, 10]                                 # planted ties: rows equal to codeword 10 take 10
    X = r.standard_normal((n, d)).astype(np.float32)
    X[:50] = CBs[:, 10].reshape(-1)
    codes = torch.empty((M, n), dtype=torch.uint8, device=DEV)
    x, lab, c, cb0 = _t(X), _t(np.zeros(n, np.int64)), _t(C), _t(CBs)
    lib.call("dirb200_pq_assign", ops._ptr(x), n, d, ops._ptr(lab), ops._ptr(c), ops._ptr(cb0), M, ops._ptr(codes), 1,
             ops._stream())
    want = P.encode(X, CBs)
    assert np.array_equal(codes.cpu().numpy().T, want) and (want[:50] == 10).all()
    cb = _t(CBs)
    empty = torch.zeros(1, dtype=torch.int64, device=DEV)
    lib.call("dirb200_pq_update", ops._ptr(x), n, d, ops._ptr(lab), ops._ptr(c), ops._ptr(codes), M, ops._ptr(cb),
             ops._ptr(empty), ops._stream())
    wcb, wempty = P.update(X, want, CBs)
    assert np.array_equal(cb.cpu().numpy(), wcb) and int(empty) == wempty
    assert np.array_equal(cb.cpu().numpy()[:, 11], CBs[:, 11])      # no member: kept


@pytest.fixture(scope="module")
def built():
    ivfpq, ivf, ops, _ = _mods()
    X, C, q = _data(20000, 64, 7, 30, seed=1)
    index = ivfpq.IVFPQIndex(_t(X), _t(C), 16, train_size=1000, pq_iter=3, seed=0)
    labels, perm, off = _model_lists(X, C)
    CBs, _ = P.train(X, C, labels, 16, 1000, 3, 0)
    codes = P.encode(P.residuals(X, C, labels), CBs)[perm]
    yield dict(index=index, X=X, C=C, q=q, perm=perm, off=off, T=P.tables(q, CBs), codes=codes,
               E=KM.exact_scores(q, X), Ec=KM.exact_scores(q, C))
    index.close()


# (1, 10, 310): query 29 has rows 5 and 11 (equal codes, equal ADC scores) at positions 310 and 311, so the R-th key is
# decided by the row bits
@pytest.mark.parametrize("nprobe,k,R", [(1, 10, 10), (2, 10, 40), (3, 50, 200), (6, 1, 3000), (2, 100, 100),
                                        (1, 10, 310)])
def test_search_equals_model(built, nprobe, k, R):
    b = built
    assert np.array_equal(b["codes"], b["index"].codes_.cpu().numpy())
    probes = b["index"].probe(_t(b["q"]), nprobe).cpu().numpy()
    assert np.array_equal(probes, IM.probe(b["Ec"], nprobe))
    sc, ix, cands = P.search(b["E"], b["T"], b["Ec"], probes, b["codes"], b["perm"], b["off"], k, R)
    s, i = b["index"].search(_t(b["q"]), k, nprobe, refine=R)
    assert np.array_equal(i.cpu().numpy(), ix) and np.array_equal(s.cpu().numpy(), sc)
    # C_q itself: a search as deep as R returns all of it in exact order
    _, i = b["index"].search(_t(b["q"]), R, nprobe, refine=R)
    for qi, cq in enumerate(cands):
        got = i.cpu().numpy()[qi]
        assert sorted(got[got >= 0].tolist()) == sorted(cq.tolist())


@pytest.mark.parametrize("nq,nprobe", [(300, 7), (600, 7), (1000, 3)])
def test_probe_groups_equal_model(built, nq, nprobe):
    """Q * nprobe >= 2048: the scan gives each CTA a group of probes (2, 4 and 2 here; 7 probes in groups of 4 leave an
    uneven last group), and a CTA past the first group starts its segment after the earlier probes' rows."""
    b = built
    r = np.random.RandomState(nq)
    q = _unit(b["X"][r.randint(0, b["X"].shape[0], nq)] + 0.3 * r.standard_normal((nq, 64)))
    Ec, E = KM.exact_scores(q, b["C"]), KM.exact_scores(q, b["X"])
    probes = IM.probe(Ec, nprobe)
    T = P.tables(q, b["index"].codebooks_.cpu().numpy())
    sc, ix, _ = P.search(E, T, Ec, probes, b["codes"], b["perm"], b["off"], 10, 50)
    s, i = b["index"].search(_t(q), 10, nprobe, refine=50)
    assert np.array_equal(i.cpu().numpy(), ix) and np.array_equal(s.cpu().numpy(), sc)


@pytest.mark.parametrize("k", [1, 100, 5000])
def test_full_refine_equals_ivf_and_exact_search(k):
    ivfpq, ivf, ops, _ = _mods()
    X, C, q = _data(30000, 2048, 9, 12, seed=4)
    pq = ivfpq.IVFPQIndex(_t(X), _t(C), 64, train_size=2000, pq_iter=2)
    lists = ivf.IVFIndex(_t(X), _t(C))
    exact = ops.Index(_t(X))
    try:
        for nprobe in (1, 4):
            a = pq.search(_t(q), k, nprobe, refine=30000)
            b = lists.search(_t(q), k, nprobe)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        a = pq.search(_t(q), k, 9, refine=30000)
        b = exact.search(_t(q), k)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    finally:
        pq.close()
        lists.close()
        exact.close()


def test_chunked_and_host_builds_equal_one_shot():
    ivfpq, _, _, lib = _mods()
    X, C, q = _data(10000, 2048, 6, 20, seed=5)
    one = ivfpq.IVFPQIndex(_t(X), _t(C), 32, train_size=800, pq_iter=2)
    chunked = ivfpq.IVFPQIndex(_t(X), _t(C), 32, train_size=800, pq_iter=2, chunk_rows=3334)
    host = ivfpq.IVFPQIndex(X, C, 32, train_size=800, pq_iter=2, chunk_rows=4000, rows="host")
    try:
        assert chunked.chunks_ == 3 and host.chunks_ == 3 and not host.rows_.is_cuda and host.rows_.is_pinned()
        for other in (chunked, host):
            assert torch.equal(one.codes_, other.codes_) and torch.equal(one.codebooks_, other.codebooks_)
        assert host.device_bytes_ < one.device_bytes_ - X.nbytes + 1
        for nprobe, R in ((2, 40), (6, 10000)):
            a, b = one.search(_t(q), 20, nprobe, refine=R), host.search(_t(q), 20, nprobe, refine=R)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        host.rows_ = host.rows_.clone()                      # pageable: refused
        assert not host.rows_.is_pinned()
        with pytest.raises(lib.DirbError):
            host.search(_t(q), 5, 2)
    finally:
        one.close()
        chunked.close()
        host.close()


def test_deterministic_across_runs_blocks_and_budgets(built):
    idx, q = built["index"], _t(built["q"])
    ref = idx.search(q, 30, 3, refine=120)
    for budget in (1 << 30, 300000, 1):
        idx.set_option("ws_budget", budget)
        got = idx.search(q, 30, 3, refine=120)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
        if budget == 1:
            assert idx.stats()["blocks"] == q.shape[0]
    idx.set_option("ws_budget", 1 << 30)
    idx.set_option("profile", 1)
    got = idx.search(q, 30, 3, refine=120)
    idx.set_option("profile", 0)
    st = idx.stats()
    assert torch.equal(got[1], ref[1]) and st["segments"] == q.shape[0] * 3 and st["scan_ms"] >= 0
    assert st["candidates"] == sum(min(120, len(IM.union(p, built["perm"], built["off"])))
                                   for p in IM.probe(built["Ec"], 3))


def test_rank_counts_equal_model(built):
    _, _, ops, _ = _mods()
    b = built
    r = np.random.RandomState(7)
    off = np.arange(0, 31 * 8, 8, dtype=np.int64)
    t_rows = r.randint(0, 20000, 30 * 8).astype(np.int64)
    flags = np.ones(t_rows.shape[0], np.uint8)
    flags[::5] = 0
    exact = ops.Index(_t(b["X"]))
    try:
        for nprobe, R in ((2, 50), (4, 400), (7, 20000)):
            inside, sc, rank = b["index"].rank_counts(_t(b["q"]), off, t_rows, flags, nprobe, refine=R, exact=exact)
            probes = IM.probe(b["Ec"], nprobe)
            _, _, cands = P.search(b["E"], b["T"], b["Ec"], probes, b["codes"], b["perm"], b["off"], 1, R)
            t_q = np.repeat(np.arange(30), 8)
            want = np.where(flags != 0, P.ranks(b["E"], cands, t_q, t_rows), 0)
            assert np.array_equal(rank.cpu().numpy(), want)
            assert np.array_equal(inside.cpu().numpy(), [t in set(cands[qq].tolist()) for qq, t in zip(t_q, t_rows)])
    finally:
        exact.close()


def test_errors(built):
    ivfpq, _, _, _ = _mods()
    X, C, q = built["X"], built["C"], _t(built["q"])
    idx = built["index"]
    for kw in (dict(k=0, nprobe=1), dict(k=5, nprobe=0), dict(k=5, nprobe=8), dict(k=5, nprobe=1, refine=4),
               dict(k=5, nprobe=1, refine=0)):
        with pytest.raises(ValueError):
            idx.search(q, **kw)
    with pytest.raises(ValueError):
        idx.search(q * 2, 5, 1)
    for M in (7, 256, 48):
        with pytest.raises(ValueError):
            ivfpq.IVFPQIndex(_t(X), _t(C), M)
    with pytest.raises(ValueError):
        ivfpq.IVFPQIndex(_t(X * 1.5), _t(C), 8)
    with pytest.raises(ValueError):
        ivfpq.IVFPQIndex(_t(X[:200]), _t(C), 8)              # fewer than 256 training rows
    with pytest.raises(ValueError):
        ivfpq.IVFPQIndex(_t(X), _t(C), 8, rows="disk")


def test_train_fits_the_ivf_lists():
    ivfpq, ivf, _, _ = _mods()
    X, _, q = _data(5000, 64, 8, 5, seed=8)
    pq = ivfpq.IVFPQIndex.train(_t(X), 8, 16, pq_iter=1)
    lists = ivf.IVFIndex.train(_t(X), 8)
    try:
        assert torch.equal(pq.centres_, lists.centres_) and torch.equal(pq.perm_, lists.perm_)
        assert torch.equal(pq.probe(_t(q), 3), lists.probe(_t(q), 3))
    finally:
        pq.close()
        lists.close()
    # a host array larger than fit_rows: the lists are fitted on the sorted sample default_rng(seed) draws
    from dirb200.cluster import SphericalKMeans
    pq = ivfpq.IVFPQIndex.train(X, 8, 16, fit_rows=2000, pq_iter=1, chunk_rows=1500)
    try:
        sel = np.sort(np.random.default_rng(0).choice(5000, 2000, replace=False))
        km = SphericalKMeans(8, init="k-means++", max_iter=20, seed=0).fit(_t(X[sel]))
        assert torch.equal(pq.centres_, km.cluster_centers_)
    finally:
        pq.close()


def _p8_aps(qd, bd, gnd, nprobe, R, M):
    """Rule P8's list L_q from the numpy model on the descriptors the grading received, junk removed, AP of the
    positives.  The lists and codebooks are IVFPQIndex.train's on those rows (deterministic: the same as the grading's)."""
    from dirb200.datasets import compute_average_precision
    from dirb200.ivfpq import IVFPQIndex
    idx = IVFPQIndex.train(_t(bd), 4, M)
    T = P.tables(qd, idx.codebooks_.cpu().numpy())
    codes, perm, off = idx.codes_.cpu().numpy(), idx.perm_.cpu().numpy(), idx.cell_off_.cpu().numpy()
    C = idx.centres_.cpu().numpy()
    idx.close()
    n = bd.shape[0]
    E, Ec = KM.exact_scores(qd, bd), KM.exact_scores(qd, C)
    _, _, cands = P.search(E, T, Ec, IM.probe(Ec, nprobe), codes, perm, off, 1, R)
    aps = []
    for qi, g in enumerate(gnd):
        cq = set(cands[qi].tolist())
        junk = set(g["junk"])
        order = [r for r in sorted(range(n), key=lambda r: (r not in cq, -E[qi, r], r)) if r not in junk]
        rank = {r: i for i, r in enumerate(order)}
        aps.append(compute_average_precision(np.sort([rank[p] for p in g["ok"]])))
    return aps


def test_dir_main_with_pq(tmp_path, monkeypatch):
    """test_dir --ivf --pq on the synthetic Oxford layout (with enough unlabelled images for 256 training rows): R at
    least every probed row gives the APs of plain --ivf; a small R gives the APs of the numpy model of rule P8 on the
    descriptors the grading receives (after --aqe, or --whiten); both with and without --aqe / --whiten."""
    _mods()
    import e2e_data
    from sklearn.decomposition import PCA
    from dirb200 import pipeline
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root, hard=True, n_extra=300)
    ckpt = os.path.join(root, "ckpt.pt")
    opts = dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_options": opts}, ckpt)
    monkeypatch.setenv("DB_ROOT", root)
    from dirtorch import test_dir
    saved = os.path.join(root, "saved")
    base = ["--dataset", "Oxford5K", "--checkpoint", ckpt, "--whiten", "", "--gpu", "0", "--threads", "2", "--detailed"]
    test_dir.test_dir_main(base + ["--save-feats", saved])
    B = np.load(os.path.join(saved, "feats.bdescs.npy"))
    load = base + ["--load-feats", saved]
    n = B.shape[0]
    pca = PCA(n_components=64, whiten=True).fit(B)
    ckpt_w = os.path.join(root, "ckpt_w.pt")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_options": opts, "pca": {"W": pca}}, ckpt_w)
    wl = ["--dataset", "Oxford5K", "--checkpoint", ckpt_w, "--whiten", "W", "--gpu", "0", "--load-feats", saved, "--detailed"]
    seen = []
    orig = pipeline._aps_from_ivf

    def record(db, qdescs, bdescs, params):
        seen.append((qdescs.cpu().numpy(), bdescs.cpu().numpy()))
        return orig(db, qdescs, bdescs, params)

    monkeypatch.setattr(pipeline, "_aps_from_ivf", record)
    for argv, M in ((load, 32), (load + ["--aqe", "2", "1"], 32), (wl, 8), (wl + ["--aqe", "2", "1"], 8)):
        for nprobe in (1, 2):
            plain = test_dir.test_dir_main(argv + ["--ivf", "4", str(nprobe)])
            full = test_dir.test_dir_main(argv + ["--ivf", "4", str(nprobe), "--pq", str(M), "--refine", str(n)])
            assert full["APs"] == plain["APs"]
        seen.clear()
        r = test_dir.test_dir_main(argv + ["--ivf", "4", "2", "--pq", str(M), "--refine", "10"])
        (qd, bd), = seen
        np.testing.assert_allclose(r["APs"], _p8_aps(qd, bd, gnd, 2, 10, M), rtol=0, atol=1e-12)
