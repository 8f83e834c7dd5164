"""Range search, triangular self-join and duplicate groups on the GPU (DESIGN.md section 4.8, rules J1-J6).  -m gpu

range_search(q, tau) must equal, bit for bit, the prefix of the exact ranking Index.search(q, N) down to its last
score >= tau; self_join(tau) must equal range_search(X, tau) without the entries j <= i; the labels must equal
scipy's components relabelled by their smallest row.  Band edges come from tests/band_data.py."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from scipy.sparse.csgraph import connected_components

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import band_data as B  # noqa: E402
import join_model as JM  # noqa: E402
import search_model as SM  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _rows(N, D, seed=0, dup_every=50):
    """Clustered unit rows (within-cluster scores ~0.85), every dup_every-th row a copy of the one before."""
    r = np.random.RandomState(seed)
    k = max(1, N // 10)
    c = r.standard_normal((k, D)).astype(np.float32)
    X = c[r.randint(0, k, N)] + 0.3 * r.standard_normal((N, D)).astype(np.float32)
    X[dup_every::dup_every] = X[dup_every - 1:-1:dup_every][: X[dup_every::dup_every].shape[0]]
    return (X / np.linalg.norm(X, axis=1, keepdims=True)).astype(np.float32)


def _np(res):
    return tuple(t.cpu().numpy() for t in res)


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def _check_range(idx, q, tau):
    """range_search == the prefix of the exact ranking with score >= tau (rows and fp64 bits)."""
    off, rows, sc = _np(idx.range_search(q, tau))
    s, i = (t.cpu().numpy() for t in idx.search(q, idx.n))
    assert off[0] == 0 and len(off) == q.shape[0] + 1
    for qi in range(q.shape[0]):
        k = int((s[qi] >= tau).sum())
        assert np.array_equal(rows[off[qi]:off[qi + 1]], i[qi, :k]), (qi, tau)
        assert np.array_equal(_bits(sc[off[qi]:off[qi + 1]]), _bits(s[qi, :k])), (qi, tau)
    return off, rows, sc


def _without_lower(off, rows, sc):
    n = len(off) - 1
    keep = rows > np.repeat(np.arange(n), np.diff(off))
    cum = np.concatenate([[0], np.cumsum(keep)])
    return cum[off].astype(np.int64), rows[keep], sc[keep]


def _same(a, b):
    return all(np.array_equal(np.asarray(x).view(np.int64) if np.asarray(x).dtype == np.float64 else np.asarray(x),
                              np.asarray(y).view(np.int64) if np.asarray(y).dtype == np.float64 else np.asarray(y))
               for x, y in zip(a, b))


def _check_self(idx, X, tau, row_block=None):
    got = _np(idx.self_join(tau, row_block=row_block))
    want = _without_lower(*_np(idx.range_search(X, tau)))
    assert _same(got, want), (tau, row_block)
    return got


def _scipy_labels(off, cols, n):
    g = sp.csr_matrix((np.ones(len(cols)), cols, off), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    first = {}
    for i, l in enumerate(lab):
        first.setdefault(l, i)
    return np.array([first[l] for l in lab], np.int64)


# ------------------------------------------------------------------------------------------------ range search
@pytest.mark.parametrize("D", [64, 2048])
@pytest.mark.parametrize("N", [1, 2, 127, 128, 129, 4097, 20000])
def test_range_search_is_the_prefix_of_the_exact_ranking(N, D):
    ops = _ops()
    X = _rows(N, D, seed=N + D)
    Q = min(N, 9)
    q = _t(np.concatenate([X[:Q], _rows(3, D, seed=7)]))       # database rows (self included) and outside queries
    idx = ops.Index(_t(X))
    s = idx.search(q, N)[0].cpu().numpy()
    planted = [float(s[0, min(N - 1, 3)]), float(s[1 if Q > 1 else 0, N // 2])]    # exact scores: inclusive boundary
    for tau in [1.5, -1.0, 0.9, 0.8, 0.0] + planted:
        off, rows, sc = _check_range(idx, q, tau)
        if tau == 1.5:
            assert off[-1] == 0
    for tau in planted:
        off, _, sc = _np(idx.range_search(q, tau))
        assert (sc == tau).any()


def test_range_search_of_rows_equal_to_tau_and_duplicates():
    ops = _ops()
    X = _rows(3000, 256, seed=5, dup_every=3)                     # many exact ties between copies
    idx = ops.Index(_t(X))
    _check_range(idx, _t(X[:40]), 0.85)
    _check_range(idx, _t(X[:40]), float(idx.search(_t(X[:1]), 10)[0][0, 1]))


# ------------------------------------------------------------------------------------------------ self-join
@pytest.mark.parametrize("D", [64, 2048])
@pytest.mark.parametrize("N", [1, 2, 127, 128, 129, 4097, 20000])
def test_self_join_is_range_search_without_lower_entries(N, D):
    ops = _ops()
    X = _rows(N, D, seed=N + 2 * D)
    idx = ops.Index(_t(X))
    Xd = _t(X)
    for tau in (0.9, 0.8, 1.5):
        got = _check_self(idx, Xd, tau)
        if tau == 1.5:
            assert got[0][-1] == 0
    if N <= 4097:
        _check_self(idx, Xd, -1.0)
    if N > 256:
        base = _np(idx.self_join(0.8))
        for rb in (128, 256, 384):
            assert _same(_np(idx.self_join(0.8, row_block=rb)), base), rb


def test_self_join_all_pairs_and_duplicates():
    ops = _ops()
    N = 700
    X = _rows(N, 128, seed=1)
    idx = ops.Index(_t(X))
    off, cols, sc = _check_self(idx, _t(X), -2.0)
    assert off[-1] == N * (N - 1) // 2
    assert np.array_equal(np.diff(off), N - 1 - np.arange(N))
    Y = np.repeat(_rows(50, 128, seed=2), 6, axis=0)              # every row six times: identical rows are pairs
    idy = ops.Index(_t(Y))
    off, cols, sc = _check_self(idy, _t(Y), 0.999)
    for i in range(0, 300, 6):
        assert set(cols[off[i]:off[i + 1]]) >= set(range(i + 1, i + 6))


def test_self_join_row_block_above_zero():
    """Row ranges [row0, row1) of the C ABI: the CSR of a middle range equals the rows of the full join."""
    from dirb200 import lib
    import ctypes as C
    ops = _ops()
    X = _rows(1000, 64, seed=3)
    idx = ops.Index(_t(X))
    full = _np(idx.self_join(0.8))
    total = C.c_int64()
    lib.call("dirb200_index_self_join", idx._h, 256, 700, 0.8, C.byref(total), ops._stream())
    off, rows, sc = _np(idx._join_result(700 - 256, total.value))
    f_off, f_rows, f_sc = full
    assert np.array_equal(off, f_off[256:701] - f_off[256])
    assert np.array_equal(rows, f_rows[f_off[256]:f_off[700]])
    assert np.array_equal(_bits(sc), _bits(f_sc[f_off[256]:f_off[700]]))
    with pytest.raises(lib.DirbError):
        lib.call("dirb200_index_self_join", idx._h, 100, 700, 0.8, C.byref(total), ops._stream())
    with pytest.raises(ValueError):
        idx.self_join(0.8, row_block=100)


# ------------------------------------------------------------------------------------------------ band edges
def _band_set(D=2048, scale=1.0):
    q, up = B.band_query(D, seed=11)
    n = 24
    traps = B.planted_rows(q, up, "trap", [B.STEP * (1 + j % 3) for j in range(n)], scale=scale, seed=1)
    decoys = B.planted_rows(q, up, "decoy", [-B.STEP * (1 + j % 3) for j in range(n)], scale=scale, seed=2)
    db = np.concatenate([B.fillers(q, np.linspace(0.1, 1.0, 200), scale=scale, seed=3), traps, decoys])
    return q, db, np.arange(200, 200 + n), np.arange(200 + n, 200 + 2 * n)


def test_band_edges_range_search():
    ops = _ops()
    q, db, trp, dec = _band_set()
    ex = SM.exact_scores(q[None], db)[0]
    fast = SM.fast_scores(q[None], db)[0]
    assert np.all(ex[trp] > 0) and np.all(ex[dec] < 0)
    assert np.all(fast[trp] < 0) and np.all(fast[dec] > 0)      # the fp16 path orders them the other way round
    idx = ops.Index(_t(db), check_norms=False)
    off, rows, sc = _check_range(idx, _t(q[None]), 0.0)
    assert set(rows.tolist()) == set(trp.tolist())               # every trap reported, no decoy
    gap = float(fast[dec].min() - fast[trp].max())
    idx.set_option("eps16", 0.45 * gap)                          # a band narrower than the traps' deficit
    off2, rows2, _ = _np(idx.range_search(_t(q[None]), 0.0))
    assert len(rows2) < len(trp)
    # the self-join of the query with the planted rows: the query's partners are exactly the traps
    X = np.concatenate([q[None], db]).astype(np.float32)
    idj = ops.Index(_t(X), check_norms=False)
    off, cols, sc = _check_self(idj, _t(X), 0.0)
    assert set(cols[off[0]:off[1]].tolist()) == set((trp + 1).tolist())


def test_band_edges_non_unit_rows():
    ops = _ops()
    scale = 4.0
    q, db, trp, dec = _band_set(scale=scale)
    idx = ops.Index(_t(db), check_norms=False)
    qn, rn = float(np.linalg.norm(q)), float(np.linalg.norm(db, axis=1).max())
    idx.set_option("eps16", B.unnormalised_eps16(qn, rn, q.shape[0]))
    off, rows, sc = _check_range(idx, _t(q[None]), 0.0)
    assert set(rows.tolist()) == set(trp.tolist())


# ------------------------------------------------------------------------------------------------ completeness
def test_overflow_capacity_blocks_and_determinism():
    ops = _ops()
    X = _rows(5000, 128, seed=9, dup_every=4)
    idx = ops.Index(_t(X))
    q = _t(X[:300])
    base_r = _np(idx.range_search(q, 0.8))
    base_s = _np(idx.self_join(0.8))
    assert _same(_np(idx.range_search(q, 0.8)), base_r) and _same(_np(idx.self_join(0.8)), base_s)
    idx.set_option("join_cap", 1)                                # every list overflows: re-runs at the exact count
    assert _same(_np(idx.range_search(q, 0.8)), base_r)
    assert _same(_np(idx.self_join(0.8)), base_s)
    assert idx.join_stats()["reruns"] >= 1
    idx.set_option("ws_budget", 600_000)                         # small blocks, halved on overflow
    assert _same(_np(idx.range_search(q, 0.8)), base_r)
    assert _same(_np(idx.self_join(0.8)), base_s)
    assert idx.join_stats()["filter_launches"] > 4
    idx.set_option("join_cap", 0)
    idx.set_option("ws_budget", 20_000)                          # cannot hold one row's candidates: a clear error
    from dirb200 import lib
    with pytest.raises(lib.DirbError, match="candidates"):
        idx.range_search(q, -1.0)


# ------------------------------------------------------------------------------------------------ components
def _csr(n, pairs):
    pairs = sorted(pairs)
    off = np.zeros(n + 1, np.int64)
    for i, _ in pairs:
        off[i + 1] += 1
    return np.cumsum(off), np.array([j for _, j in pairs], np.int64)


@pytest.mark.parametrize("case", ["chain", "star", "star_last", "clique", "isolated", "one", "random"])
def test_components_match_scipy(case):
    ops = _ops()
    r = np.random.RandomState(0)
    n, pairs = {
        "chain": (10000, [(i, i + 1) for i in range(9999)]),
        "star": (5000, [(0, j) for j in range(1, 5000)]),
        "star_last": (5000, [(i, 4999) for i in range(4999)]),
        "clique": (300, [(i, j) for i in range(300) for j in range(i + 1, 300)]),
        "isolated": (1000, []),
        "one": (1, []),
        "random": (3000, sorted({tuple(sorted(p)) for p in r.randint(0, 3000, (2500, 2)) if p[0] != p[1]})),
    }[case]
    off, cols = _csr(n, pairs)
    labels = ops.join_components(_t(off), _t(cols), n).cpu().numpy()
    assert np.array_equal(labels, _scipy_labels(off, cols, n))
    goff, mem = (t.cpu().numpy() for t in ops.join_groups(_t(labels)))
    want = JM.groups(labels)
    assert len(goff) - 1 == len(want)
    for g, w in enumerate(want):
        assert np.array_equal(mem[goff[g]:goff[g + 1]], w)


def test_near_duplicates_on_its_own_pairs():
    from dirb200 import duplicates as DU
    X = _rows(6000, 256, seed=4, dup_every=7)
    d = DU.near_duplicates(X, 0.9)
    off, cols = d.off.cpu().numpy(), d.cols.cpu().numpy()
    labels = d.labels.cpu().numpy()
    assert np.array_equal(labels, _scipy_labels(off, cols, 6000))
    assert [list(g) for g in JM.groups(labels)] == d.group_lists()
    d2 = DU.near_duplicates(_t(X), 0.9, row_block=1024)
    assert all(_same(_np((a,)), _np((b,))) for a, b in zip(d[:4], d2[:4]))
    with pytest.raises(ValueError):
        DU.near_duplicates(2 * X, 0.9)                                  # not unit-norm and no eps16
    with pytest.raises(ValueError):
        DU.overlap(X[:, :128], X, 0.9)
    o = _np(DU.overlap(X[:50], X, 0.9))
    idx = _ops().Index(_t(X))
    assert _same(o, _np(idx.range_search(_t(X[:50]), 0.9)))


# ------------------------------------------------------------------------------------------------ command line
def test_find_duplicates_end_to_end(tmp_path, monkeypatch, capsys):
    """The planted copy groups of the synthetic Oxford layout, from --load-feats and from --dataset images, and the
    planted overlap of two sets with --against."""
    import json
    import e2e_data
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "model_options": dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)},
               os.path.join(root, "ckpt.pt"))
    monkeypatch.setenv("DB_ROOT", root)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    dataset = 'ImageList("%s/list.txt", "%s/oxford5k/jpg")' % (root, root)
    from dirtorch import extract_features, find_duplicates
    feats_npy = os.path.join(root, "feats.npy")
    extract_features.extract_features_main(["--dataset", dataset, "--checkpoint", os.path.join(root, "ckpt.pt"),
                                            "--output", feats_npy, "--gpu", "0", "--threads", "2"])
    F = np.load(feats_npy)
    planted = [list(range(4 * g, 4 * g + 4)) for g in range(8)]        # each image and its three noisy copies
    E = F.astype(np.float64) @ F.astype(np.float64).T
    same = np.zeros_like(E, bool)
    for g in planted:
        same[np.ix_(g, g)] = True
    np.fill_diagonal(same, False)
    lo, hi = E[same].min(), E[~same & ~np.eye(len(F), dtype=bool)].max()
    assert lo > hi + 1e-4, (lo, hi)                                      # the layout separates the copies
    tau = float((lo + hi) / 2)
    out = os.path.join(root, "dups.npz")
    res = find_duplicates.find_duplicates_main(["--load-feats", feats_npy, "--threshold", repr(tau), "--output", out])
    assert res["groups"] == planted
    z = np.load(out)
    assert len(z["pairs"]) == 8 * 6 and set(z.files) == {"pairs", "scores", "labels"}
    assert "%d rows: 48 pairs" % len(F) in capsys.readouterr().out
    js = os.path.join(root, "groups.json")
    res2 = find_duplicates.find_duplicates_main(["--dataset", dataset, "--checkpoint", os.path.join(root, "ckpt.pt"),
                                                 "--threshold", repr(tau), "--out-json", js, "--threads", "2"])
    assert res2["groups"] == planted
    assert json.load(open(js))["groups"] == [[names[i] for i in g] for g in planted]
    # --against: the originals of groups 0-3 against the copies of every group
    a_npy, b_npy = os.path.join(root, "a.npy"), os.path.join(root, "b.npy")
    orig = [4 * g for g in range(4)]
    copies = [i for g in planted for i in g[1:]]
    np.save(a_npy, F[orig])
    np.save(b_npy, F[copies])
    res3 = find_duplicates.find_duplicates_main(["--load-feats", a_npy, "--against", b_npy, "--threshold", repr(tau)])
    want = sorted((a, copies.index(c)) for a, o in enumerate(orig) for c in range(o + 1, o + 4))
    assert sorted(map(tuple, res3["pairs"].tolist())) == want
