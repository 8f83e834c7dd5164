"""Host side of the GPU PCA fit: the finalisation (n, sums, Gram) -> sklearn PCA against sklearn's own fit, the input
checks, the learn_whiten command line, and the Gram model's planted bugs against the per-element bound."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import REPO

sys.path.insert(0, os.path.join(REPO, "tests"))
import pca_model as M  # noqa: E402


def _stats(x64):
    s = x64.sum(0)
    a = x64 - s / x64.shape[0]
    return s, a.T @ a


def _spectrum(k, cluster=False):
    lam = np.geomspace(1.0, 1e-4, k)                  # gaps >= 1 % for k up to ~900
    if cluster and k > 6:
        lam[5] = lam[4]                               # an exactly repeated eigenvalue: compared through its projector
    return lam


def _compare(ours, ref, n, d, full_rank_deficient=False):
    k = ours.n_components_
    assert k == ref.n_components_ and ours.n_samples_ == n and ours.n_features_in_ == d
    np.testing.assert_allclose(ours.mean_, ref.mean_, rtol=1e-13, atol=1e-15)
    lmax = float(ref.explained_variance_[0])
    # eigenvalues within 1e-10 relative + 1e-14 lambda_max; the singular values through their squares (a numerically
    # zero eigenvalue of a rank-deficient fit is ~1e-16, its square root is not small)
    for a, b in ((ours.explained_variance_, ref.explained_variance_),
                 (ours.singular_values_ ** 2 / (n - 1), ref.singular_values_ ** 2 / (n - 1))):
        assert np.all(np.abs(a - b) <= 1e-10 * np.abs(b) + 1e-14 * lmax)
    np.testing.assert_allclose(ours.explained_variance_ratio_, ref.explained_variance_ratio_, rtol=1e-10, atol=1e-14)
    if full_rank_deficient:
        # the 'full' solver averages the discarded variance over min(n, d) values, covariance_eigh over all d
        if k < min(n, d):
            assert abs(ours.noise_variance_ * (d - k) - ref.noise_variance_ * (n - k)) <= 1e-10 * lmax
    else:
        assert abs(ours.noise_variance_ - ref.noise_variance_) <= 1e-10 * abs(ref.noise_variance_) + 1e-14 * lmax
    # components: one by one where the eigenvalue is separated from its neighbours (relative gap > 1e-4), through the
    # projector of a cluster (the repeated planted eigenvalue, split by the fp32 rounding of the data)
    lam = np.asarray(ref.explained_variance_)
    tol = 1e-12 * lmax
    i = 0
    while i < k:
        j = i + 1
        while j < k and abs(lam[j] - lam[j - 1]) <= 1e-4 * lam[j - 1]:
            j += 1
        if lam[i] <= tol:                             # the null space (n <= d): no defined direction
            break
        if j == i + 1:
            np.testing.assert_allclose(ours.components_[i], ref.components_[i], rtol=0, atol=1e-9)
        else:
            po = ours.components_[i:j].T @ ours.components_[i:j]
            pr = ref.components_[i:j].T @ ref.components_[i:j]
            np.testing.assert_allclose(po, pr, rtol=0, atol=1e-9)
        i = j


@pytest.mark.parametrize("solver", ["full", "covariance_eigh"])
@pytest.mark.parametrize("n,d", [(600, 48), (30, 48)])
@pytest.mark.parametrize("n_components", [None, 1, 32, "min"])
def test_finalisation_matches_sklearn(solver, n, d, n_components):
    from sklearn.decomposition import PCA
    from dirb200.whitening import pca_from_gram
    if n_components == "min":
        n_components = min(n, d)
    if n_components is not None and n_components > min(n, d):
        pytest.skip("more components than min(n, d)")
    lam = _spectrum(min(n - 1, d), cluster=True)
    x, _ = M.planted(n, d, lam, mean=np.linspace(-0.3, 0.5, d), seed=n + d)
    x64 = x.astype(np.float64)
    s, g = _stats(x64)
    ours = pca_from_gram(n, s, g, n_components)
    ref = PCA(n_components=n_components, whiten=True, svd_solver=solver).fit(x64)
    assert type(ours) is PCA and ours.whiten and ours.svd_solver == "covariance_eigh"
    assert ours.n_components == n_components
    for name in ("mean_", "components_", "explained_variance_", "explained_variance_ratio_", "singular_values_"):
        assert getattr(ours, name).dtype == np.float64
    _compare(ours, ref, n, d, full_rank_deficient=(solver == "full" and n < d))
    # sklearn's own transform works on the object and agrees with the reference fit on separated components
    t_ours, t_ref = ours.transform(x64[:5]), ref.transform(x64[:5])
    assert t_ours.shape == t_ref.shape


def test_sign_rule_first_index_wins_ties():
    """svd_flip(u_based_decision=False): the entry of largest |value| of every component is positive; of two equal
    magnitudes the first index decides.  The covariance below has eigenvectors (1, 1) / sqrt 2 and (1, -1) / sqrt 2."""
    from sklearn.decomposition import PCA
    from dirb200.whitening import pca_from_gram
    base = np.array([[1.0, 1.0], [-1.0, -1.0], [0.5, -0.5], [-0.5, 0.5]] * 3)
    s, g = _stats(base)
    ours = pca_from_gram(base.shape[0], s, g)
    ref = PCA(whiten=True, svd_solver="covariance_eigh").fit(base)
    for c in ours.components_:
        m = np.abs(c).max()
        first = int(np.argmax(np.abs(c)))
        assert c[first] > 0 and c[first] == m
    # sklearn's fit of the same data makes the same choice wherever its two magnitudes tie as well
    for co, cr in zip(ours.components_, ref.components_):
        if abs(cr[0]) == abs(cr[1]):
            assert np.array_equal(np.sign(co), np.sign(cr))
        np.testing.assert_allclose(co, cr, rtol=0, atol=1e-15)


def test_sign_of_largest_entry_is_positive_on_random_data():
    from dirb200.whitening import pca_from_gram
    x = np.random.RandomState(1).standard_normal((200, 20))
    s, g = _stats(x)
    p = pca_from_gram(200, s, g)
    idx = np.argmax(np.abs(p.components_), axis=1)
    assert np.all(p.components_[np.arange(20), idx] > 0)


def test_input_errors():
    from dirb200.whitening import fit_pca, pca_from_gram
    x = np.random.RandomState(2).standard_normal((10, 6))
    s, g = _stats(x)
    with pytest.raises(ValueError):
        pca_from_gram(1, x[0], np.zeros((6, 6)))
    with pytest.raises(ValueError):
        fit_pca(x[:1])                                # N < 2, refused before any device work
    for bad in (0, -1, 7, 1.5, "mle", True, 0.9):
        with pytest.raises(ValueError):
            pca_from_gram(10, s, g, bad)
        with pytest.raises(ValueError):
            fit_pca(x, n_components=bad)
    for v in (np.nan, np.inf):
        s2 = s.copy()
        s2[3] = v
        with pytest.raises(ValueError):
            pca_from_gram(10, s2, g)
    assert pca_from_gram(10, s, g, 6).n_components_ == 6 and pca_from_gram(10, s, g).n_components_ == 6


def test_learn_whiten_argument_errors(tmp_path, capsys):
    from dirb200.pipeline import learn_whiten_main
    ck = str(tmp_path / "ck.pt")
    base = ["--checkpoint", ck, "--name", "W", "--output", str(tmp_path / "out.pt")]
    with pytest.raises(SystemExit):
        learn_whiten_main(base)                                                        # no source
    with pytest.raises(SystemExit):
        learn_whiten_main(base + ["--load-feats", "a.npy", "--store", "dir"])        # two sources
    with pytest.raises(SystemExit):
        learn_whiten_main(["--checkpoint", ck, "--name", "W", "--output", ck, "--load-feats", "a.npy"])
    err = capsys.readouterr().err
    assert "exactly one of --dataset, --load-feats and --store" in err and "--output must differ" in err


def test_merge_pca_keeps_and_replaces_entries():
    from dirb200.pipeline import merge_pca
    ck = {"state_dict": {"w": torch.zeros(1)}, "pca": {"Landmarks_clean": "old", "Other": "keep"}}
    out, replaced = merge_pca(ck, "Mine", "new")
    assert not replaced and out["pca"] == {"Landmarks_clean": "old", "Other": "keep", "Mine": "new"}
    assert ck["pca"] == {"Landmarks_clean": "old", "Other": "keep"}           # the input is not modified
    out2, replaced2 = merge_pca(out, "Landmarks_clean", "newer")
    assert replaced2 and out2["pca"]["Landmarks_clean"] == "newer" and out2["pca"]["Other"] == "keep"
    out3, replaced3 = merge_pca({"state_dict": {}}, "W", "p")
    assert not replaced3 and out3["pca"] == {"W": "p"}


def test_gram_split_rule():
    assert M.gram_splits(1, 4) == (1, 32)
    assert M.gram_splits(5063, 2048) == (4, 1280)
    s, rows = M.gram_splits(1000000, 2048)
    assert s == 15 and rows % 32 == 0 and (s - 1) * rows < 1000000 <= s * rows
    t = -(-8064 // 128)
    assert t * (t + 1) // 2 <= M.GRAM_MAX_TILES < (t + 1) * (t + 2) // 2


@pytest.mark.parametrize("bug", ["drop_kstep", "mirror_transposed", "lose_last_split", "mean_fp32"])
def test_gram_bound_catches_planted_bugs(bug):
    """The model of the kernel stays within the per-element bound; each planted mistake leaves it."""
    r = np.random.RandomState(5)
    n, d = 2500, 260                                  # 3 x 3 tiles (6 computed), 2 splits, a partial last K step
    assert M.gram_splits(n, d)[0] == 2
    x = (100.0 + 1e-2 * r.standard_normal((n, d))).astype(np.float32)
    if bug == "mirror_transposed":                    # a full 128 x 128 off-diagonal tile needs d >= 256
        x = (0.1 * r.standard_normal((n, d)) + r.standard_normal(d)).astype(np.float32)
    mean = x.astype(np.float64).sum(0) / n
    g_ref, ga = M.gram_reference(x, mean)
    bound = M.gram_bound(n, ga)
    assert M.worst_ratio(M.gram_model(x, mean), g_ref, bound) <= 1.0
    assert M.worst_ratio(M.gram_model(x, mean, bug=bug), g_ref, bound) > 1.0


def test_uncentred_formula_leaves_the_bound():
    """X^T X - n m m^T (sklearn's covariance_eigh) on data with mean 100 and spread 1e-2 is far outside the bound the
    centred Gram meets."""
    r = np.random.RandomState(6)
    n, d = 3000, 20
    x = (100.0 + 1e-2 * r.standard_normal((n, d))).astype(np.float32)
    x64 = x.astype(np.float64)
    mean = x64.sum(0) / n
    g_ref, ga = M.gram_reference(x, mean)
    unc = x64.T @ x64 - n * np.outer(mean, mean)
    assert M.worst_ratio(unc, g_ref, M.gram_bound(n, ga)) > 100
    assert M.worst_ratio(M.gram_model(x, mean), g_ref, M.gram_bound(n, ga)) <= 1.0
