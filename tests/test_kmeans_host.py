"""CPU checks of the spherical k-means model (tests/kmeans_model.py): its exact score restates exact_dot_warp, its rules
agree with dense restatements, each planted bug leaves a check, well-separated clusters are recovered exactly, the
command line parses and refuses bad input, and the new kernels build without spills."""
import os
import re

import numpy as np
import pytest

import kmeans_model as M
from conftest import REPO


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _clusters(n, k, dim, seed=0, spread=0.05):
    r = np.random.RandomState(seed)
    c = _unit(r.standard_normal((k, dim)))
    truth = r.randint(0, k, n)
    return _unit(c[truth] + spread * r.standard_normal((n, dim))), truth


# ------------------------------------------------------------------------------------------------ K1 / K2
@pytest.mark.parametrize("dim", [64, 192, 256, 2048])
def test_exact_scores_restate_the_warp_order(dim):
    r = np.random.RandomState(dim)
    A, B = _unit(r.standard_normal((5, dim))), _unit(r.standard_normal((3, dim)))
    E = M.exact_scores(A, B)
    for i in range(5):
        for j in range(3):
            lanes = np.zeros(32)
            for g in range(dim // 4):
                for c in range(4):
                    lanes[g % 32] += np.float64(A[i, 4 * g + c]) * np.float64(B[j, 4 * g + c])
            for o in (16, 8, 4, 2, 1):
                lanes = lanes + lanes[np.arange(32) ^ o]
            assert E[i, j] == lanes[0]
    assert np.abs(E - A.astype(np.float64) @ B.astype(np.float64).T).max() < 1e-12
    assert np.array_equal(M.exact_scores(B, A), E.T)          # e(a, b) == e(b, a) bit for bit


@pytest.mark.parametrize("k", [1, 31, 32, 33])
def test_assignment_matches_dense_argmax(k):
    X, _ = _clusters(300, max(k, 2), 64, seed=k)
    C = X[:k].copy()
    C[k // 2] = C[0]                                          # duplicated centres: the smaller index wins
    E = M.exact_scores(X, C)
    lab, sc = M.assign(E)
    for i in range(len(X)):
        best = max(E[i])
        assert lab[i] == min(c for c in range(k) if E[i, c] == best) and sc[i] == best


def test_ties_go_to_the_smallest_centre_and_the_planted_bug_does_not():
    X, _ = _clusters(50, 3, 64)
    C = np.repeat(X[:1], 4, axis=0)                           # all-equal centres
    lab, _ = M.assign(M.exact_scores(X, C))
    assert (lab == 0).all()
    bad, _ = M.assign(M.exact_scores(X, C), bug="ties_last")
    assert (bad == 3).all()



# ------------------------------------------------------------------------------------------------ K3
EPS16 = 1.2e-3


def _planted(n, k, seed, ties=None):
    """Exact scores E and fp16-path scores F anywhere within +-EPS16 of them, extremes included."""
    r = np.random.RandomState(seed)
    E = np.round(r.uniform(-0.2, 0.9, (n, k)), 3)           # coarse values: many exact ties
    if ties == "all":
        E[:] = E[:, :1]
    noise = r.choice([-1.0, 1.0, -0.999, 0.999, 0.0], (n, k)) * r.uniform(0.5, 1.0, (n, k))
    F = (E + noise * EPS16).astype(np.float32)
    F = np.clip(F, np.nextafter((E - EPS16).astype(np.float32), np.float32(np.inf)),
                np.nextafter((E + EPS16).astype(np.float32), np.float32(-np.inf)))
    return E, F


@pytest.mark.parametrize("k", [1, 31, 32, 33, 64, 100])
@pytest.mark.parametrize("ties", [None, "all"])
def test_candidate_groups_hold_the_exact_argmax(k, ties):
    for seed in range(5):
        E, F = _planted(200, k, seed, ties)
        assert (np.abs(F.astype(np.float64) - E) <= EPS16).all()
        for cap in (0, 1, 16):
            lab, sc = M.nearest(E, F, EPS16, cap)
            want, wsc = M.assign(E)
            assert np.array_equal(lab, want) and np.array_equal(sc, wsc)


def test_candidates_ties_inside_and_across_groups():
    E = np.zeros((1, 96))
    E[0, [5, 7, 40, 70]] = 0.8                                 # ties inside group 0 and across groups 1, 2
    F = (E + EPS16 * np.where(np.arange(96) == 70, 1.0, -1.0)).astype(np.float32)
    c, ng, full = M.candidates(F[0], EPS16, 16)
    assert not full and ng == 3 and {5, 7, 40, 70} <= set(c.tolist())
    assert M.nearest(E, F, EPS16)[0][0] == 5
    c, _, full = M.candidates(F[0], EPS16, 2)                  # more groups than the cap: every centre
    assert full and len(c) == 96


def test_band_threshold_rounds_down():
    r = np.random.RandomState(0)
    caught = 0
    for m, eps in zip(r.uniform(-1, 1, 2000).astype(np.float32), r.uniform(1e-4, 5e-3, 2000)):
        x = float(m) - 2.0 * float(eps)
        t = M.band_threshold(m, eps)
        assert float(t) <= x < float(np.nextafter(t, np.float32(np.inf)))
        caught += float(M.band_threshold(m, eps, bug="round_nearest")) > x
    assert caught > 500


def test_planted_band1_bug():
    # the best centre sits eps16 below its exact score, another eps16 above its slightly smaller one: a band of one
    # eps16 drops the best centre's group
    E = np.zeros((1, 64))
    E[0, 3], E[0, 40] = 0.5, 0.4995
    F = (E + EPS16 * np.where(np.arange(64) == 40, 0.99, -0.99)).astype(np.float32)
    assert M.nearest(E, F, EPS16)[0][0] == 3
    assert M.nearest(E, F, EPS16, bug="band1")[0][0] == 40

# ------------------------------------------------------------------------------------------------ K4
def _relocation_case():
    labels = np.array([0, 0, 0, 1, 3, 3, 5, 5, 5], np.int64)
    scores = np.array([0.9, 0.2, 0.5, 0.1, 0.3, 0.3, 0.8, 0.7, 0.25])
    return labels, scores, 7                                  # clusters 2, 4, 6 are empty


def test_relocation_rule():
    labels, scores, k = _relocation_case()
    out, moves = M.relocate(labels, scores, k)
    # order by (score, row): 3 (0.1, singleton: skipped), 1 (0.2) -> 2, 8 (0.25) -> 4, 4 (0.3) -> 6
    assert moves == 3
    assert out.tolist() == [0, 2, 0, 1, 6, 3, 5, 5, 4]
    assert (np.bincount(out, minlength=k) >= 1).all()


def test_relocation_updates_sizes_after_each_move():
    labels = np.array([0, 0, 1, 1, 1], np.int64)
    scores = np.array([0.1, 0.2, 0.3, 0.4, 0.5])
    out, moves = M.relocate(labels, scores, 4)                # clusters 2, 3 empty; cluster 0 can spare one row only
    assert moves == 2 and out.tolist() == [2, 0, 3, 1, 1]


def test_planted_singleton_bug():
    labels, scores, k = _relocation_case()
    bad, _ = M.relocate(labels, scores, k, bug="singleton")
    assert (np.bincount(bad, minlength=k) == 0).any() or not np.array_equal(bad, M.relocate(labels, scores, k)[0])


# ------------------------------------------------------------------------------------------------ K5
def test_centre_sum_order():
    r = np.random.RandomState(3)
    X = r.standard_normal((700, 64)).astype(np.float32) * np.float32(1e4)
    X[::7] *= np.float32(1e-6)
    members = np.arange(0, 700, 1)
    s = M.centre_sum(X, members)
    ref = np.zeros(64)
    for c0 in range(0, 700, 256):
        part = np.zeros(64)
        for i in range(c0, min(c0 + 256, 700)):
            part = part + X[i].astype(np.float64)
        ref = ref + part
    assert np.array_equal(s, ref)
    assert not np.array_equal(M.centre_sum(X, members, bug="order"), s)   # the planted order leaves a check


def test_norm2_order_and_zero_sum():
    r = np.random.RandomState(4)
    s = r.standard_normal(2048) * 10.0 ** r.randint(-8, 8, 2048)
    assert abs(M.norm2(s) - float(np.dot(s, s))) <= 1e-12 * float(np.dot(s, s))
    p = np.zeros(256)
    for j in range(2048):
        p[j % 256] = p[j % 256] + s[j] * s[j]
    for h in (128, 64, 32, 16, 8, 4, 2, 1):
        p[:h] = p[:h] + p[h:2 * h]
    assert M.norm2(s) == p[0]
    X = _unit(r.standard_normal((4, 64)))
    X[1] = -X[0]
    C = _unit(r.standard_normal((2, 64)))
    out, zero = M.update(X, np.array([0, 0, 1, 1]), C)       # cluster 0 = {x, -x}: keeps its centre
    assert zero == 1 and np.array_equal(out[0], C[0]) and not np.array_equal(out[1], C[1])


# ------------------------------------------------------------------------------------------------ K6 / K7
def test_objective_is_exact_in_any_order():
    r = np.random.RandomState(5)
    s = r.uniform(-1, 1, 10000)
    u = M.objective_units(s)
    assert u == M.objective_units(s[::-1]) == M.objective_units(r.permutation(s))
    assert abs(u / M.FIX - float(np.sum(s))) < 1e-5


def test_kmeans_pp_draws():
    X, _ = _clusters(400, 8, 64, seed=6)
    rows = M.kmeans_pp(X, 8, seed=1)
    assert len(set(rows.tolist())) == 8 and rows[0] == np.random.RandomState(1).randint(400)
    assert np.array_equal(rows, M.kmeans_pp(X, 8, seed=1))
    basis = np.repeat(np.eye(64, dtype=np.float32)[:3], 10, axis=0)   # e(x, x) = 1 exactly: no weight is left
    with pytest.raises(ValueError):
        M.kmeans_pp(basis, 4, seed=0)                        # three distinct rows, four centres


def test_planted_not_zeroed_bug():
    # rows a little short of unit norm keep a weight 2 - 2 e(x, x) > 0 unless chosen rows are zeroed: with n = k the
    # right rule draws every row once, the bug draws a row twice for some seed
    r = np.random.RandomState(7)
    X = (_unit(r.standard_normal((6, 64))) * np.float32(0.9995)).astype(np.float32)
    X[1:] = X[0]                                              # one distinct row away from the rest: tiny weights
    X[1:] = _unit(X[1:] + 1e-3 * r.standard_normal((5, 64)).astype(np.float32)) * np.float32(0.9995)
    differs = False
    for seed in range(40):
        good = M.kmeans_pp(X, 6, seed)
        assert sorted(good.tolist()) == list(range(6))
        differs |= sorted(M.kmeans_pp(X, 6, seed, bug="not_zeroed").tolist()) != list(range(6))
    assert differs


@pytest.mark.parametrize("init", ["k-means++", "random"])
def test_well_separated_clusters_are_recovered(init):
    X, truth = _clusters(600, 6, 64, seed=8, spread=0.02)
    out = M.fit(X, 6, init=init, seed=0 if init == "k-means++" else 3, max_iter=30)
    pairs = set(zip(truth.tolist(), out["labels"].tolist()))
    if init == "k-means++":
        assert len(pairs) == 6                                # a bijection between true and found clusters
    assert out["n_iter"] < 30 and np.array_equal(M.assign(M.exact_scores(X, out["centres"]))[0], out["labels"])
    assert out["objective"] == M.objective_units(out["scores"]) / M.FIX


def test_fit_with_an_empty_cluster_relocates():
    X, truth = _clusters(300, 4, 64, seed=9, spread=0.02)
    first = [int(np.nonzero(truth == c)[0][0]) for c in range(4)]
    init = np.concatenate([X[first], -X[first[:1]]])          # the last centre is nobody's nearest
    out = M.fit(X, 5, init=init, max_iter=10)
    assert out["relocations"] >= 1
    assert out["labels"].max() == 4 or out["n_iter"] == 10


def test_max_iter_ends_with_an_assignment_of_the_returned_centres():
    X, _ = _clusters(500, 10, 64, seed=10, spread=0.3)
    out = M.fit(X, 10, init="random", max_iter=1)
    assert out["n_iter"] == 1
    assert np.array_equal(M.assign(M.exact_scores(X, out["centres"]))[0], out["labels"])


# ------------------------------------------------------------------------------------------------ command line
def test_cli_parsing_and_errors():
    from dirb200 import cluster as K
    a = K.parse_args(["--load-feats", "x.npy", "--n-clusters", "16", "--output", "o.npz"])
    assert a.n_clusters == 16 and a.init == "k-means++" and a.max_iter == 20 and a.seed == 0 and a.gpu == 0
    a = K.parse_args(["--dataset", "ImageList('l.txt')", "--checkpoint", "c.pt", "--n-clusters", "4", "--init", "random",
                      "--max-iter", "5", "--seed", "3", "--whiten", "W", "--out-json", "c.json", "--gpu", "1"])
    assert a.init == "random" and a.max_iter == 5 and a.seed == 3 and a.whiten == "W" and a.gpu == 1
    assert K.parse_args(["--store", "S", "--n-clusters", "2", "--init", "c.npy"]).init == "c.npy"
    for bad in (["--load-feats", "x.npy"],                                          # no K
                ["--n-clusters", "3"],                                              # no input
                ["--load-feats", "x.npy", "--store", "S", "--n-clusters", "3"],     # two inputs
                ["--dataset", "D", "--n-clusters", "3"],                            # no checkpoint
                ["--load-feats", "x.npy", "--n-clusters", "0"],
                ["--load-feats", "x.npy", "--n-clusters", "3", "--max-iter", "-1"],
                ["--load-feats", "x.npy", "--n-clusters", "3", "--init", "bogus"]):
        with pytest.raises(SystemExit):
            K.parse_args(bad)


def test_dirtorch_exports():
    from dirtorch import cluster, cluster_features
    from dirb200 import cluster as K
    assert cluster.SphericalKMeans is K.SphericalKMeans
    assert cluster_features.cluster_features_main is K.cluster_features_main


# ------------------------------------------------------------------------------------------------ build
def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "kmeans.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    blocks = re.findall(r"Compiling entry function '(\w+kmeans_cu\w+)'.*?\n.*?\n(.*?)\n", open(log).read())
    assert len(blocks) == 10
    blocks += re.findall(r"Compiling entry function '(\w+nearest_\w+)'.*?\n.*?\n(.*?)\n",
                         open(os.path.join(os.path.dirname(log), "search.cu.log")).read())
    assert len(blocks) == 12
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
