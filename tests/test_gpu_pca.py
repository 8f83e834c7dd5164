"""The GPU PCA fit: column sums and the centred Gram element by element against numpy fp64 within their rounding
bounds (tests/pca_model.py), chunking and determinism, the fit against sklearn, the store path and the learn_whiten
command line end to end.  -m gpu."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import REPO, rel_l2

sys.path.insert(0, os.path.join(REPO, "tests"))
import pca_model as M  # noqa: E402

pytestmark = pytest.mark.gpu


def _gpu():
    from dirb200 import ops
    ops.require_gpu(0)


def _data(n, d, seed, family="generic"):
    r = np.random.RandomState(seed)
    if family == "offset":                            # |mean| >> spread: the uncentred formula cancels
        return (100.0 + 1e-2 * r.standard_normal((n, d))).astype(np.float32)
    return (r.standard_normal((n, d)) * r.uniform(0.1, 2.0, d) + r.uniform(-1, 1, d)).astype(np.float32)


def _check_stats(x, label, ratios):
    """Column sums and Gram of x on the GPU against numpy fp64, teacher-forced with the same fp64 mean."""
    from dirb200 import ops
    n, d = x.shape
    xd = torch.from_numpy(x).cuda()
    s = ops.col_sums_f64(xd).cpu().numpy()
    ref_s = x.astype(np.float64).sum(0)
    rs = M.worst_ratio(s, ref_s, M.sums_bound(x))
    mean = ref_s / n
    g = ops.gram_f64(xd, torch.from_numpy(mean).cuda()).cpu().numpy()
    g_ref, ga = M.gram_reference(x, mean)
    rg = M.worst_ratio(g, g_ref, M.gram_bound(n, ga))
    assert np.array_equal(g, g.T), label              # mirrored, not computed twice
    ratios[label] = (rs, rg)
    print("%s: sums |d|/bound %.3g, Gram |d|/bound %.3g" % (label, rs, rg))
    assert rs <= 1.0 and rg <= 1.0, label
    return g, g_ref, ga


SHAPES = [(n, d) for d in (4, 16, 48, 132) for n in (1, 7, 8191, 8193, 100000)] + \
         [(7, 2048), (8193, 2048), (100000, 2048), (7, 50), (3000, 50), (100, 132)]


def test_stats_within_bounds():
    _gpu()
    ratios = {}
    for i, (n, d) in enumerate(SHAPES):
        _check_stats(_data(n, d, seed=i), "N=%d D=%d" % (n, d), ratios)
    worst = max(max(v) for v in ratios.values())
    print("largest |d|/bound over %d shapes: %.3g" % (len(SHAPES), worst))


def test_offset_data_needs_the_centred_gram():
    """mean 100, spread 1e-2: X^T X - n m m^T (sklearn's covariance_eigh) is far outside the bound, the kernel inside."""
    _gpu()
    for n, d in ((8193, 132), (100000, 48)):
        x = _data(n, d, seed=7, family="offset")
        g, g_ref, ga = _check_stats(x, "offset N=%d D=%d" % (n, d), {})
        x64 = x.astype(np.float64)
        mean = x64.sum(0) / n
        unc = x64.T @ x64 - n * np.outer(mean, mean)
        r_unc = M.worst_ratio(unc, g_ref, M.gram_bound(n, ga))
        print("offset N=%d D=%d: uncentred formula |d|/bound %.3g" % (n, d, r_unc))
        assert r_unc > 100


def test_gram_one_million_rows():
    _gpu()
    from dirb200 import ops
    n, d = 1000000, 2048
    gen = torch.Generator(device="cuda").manual_seed(11)
    xd = (torch.randn((n, d), generator=gen, device="cuda") * 0.05 + 0.02).contiguous()
    x = xd.cpu().numpy()
    s = ops.col_sums_f64(xd).cpu().numpy()
    ref_s = np.zeros(d)
    for c in range(0, n, 100000):
        ref_s += x[c:c + 100000].astype(np.float64).sum(0)
    rs = M.worst_ratio(s, ref_s, M.sums_bound(x))
    mean = ref_s / n
    g = ops.gram_f64(xd, torch.from_numpy(mean).cuda()).cpu().numpy()
    g_ref, ga = M.gram_reference(x, mean, chunk=100000)
    rg = M.worst_ratio(g, g_ref, M.gram_bound(n, ga))
    print("N=1000000 D=2048: sums |d|/bound %.3g, Gram |d|/bound %.3g" % (rs, rg))
    assert rs <= 1.0 and rg <= 1.0


def test_chunks_and_determinism():
    _gpu()
    from dirb200 import ops
    n, d = 2500, 48
    x = _data(n, d, seed=3)
    xd = torch.from_numpy(x).cuda()
    ref_s = x.astype(np.float64).sum(0)
    mean = torch.from_numpy(ref_s / n).cuda()
    g_ref, ga = M.gram_reference(x, ref_s / n)
    whole = ops.gram_f64(xd, mean)
    assert torch.equal(whole, ops.gram_f64(xd, mean))                    # two runs: bit-identical
    assert torch.equal(ops.col_sums_f64(xd), ops.col_sums_f64(xd))
    for chunk in (1, 3, 1000):
        s = torch.zeros(d, dtype=torch.float64, device="cuda")
        g = torch.zeros((d, d), dtype=torch.float64, device="cuda")
        for c in range(0, n, chunk):
            ops.col_sums_f64(xd[c:c + chunk], s)
            ops.gram_f64(xd[c:c + chunk], mean, g)
        assert M.worst_ratio(s.cpu().numpy(), ref_s, M.sums_bound(x)) <= 1.0, chunk
        assert M.worst_ratio(g.cpu().numpy(), g_ref, M.gram_bound(n, ga)) <= 1.0, chunk


def test_abi_limits():
    _gpu()
    import ctypes as C
    from dirb200 import lib, ops
    x = torch.zeros((2, 8068), dtype=torch.float32, device="cuda")
    mean = torch.zeros(8068, dtype=torch.float64, device="cuda")
    g = torch.zeros(1, dtype=torch.float64, device="cuda")
    with pytest.raises(lib.DirbError) as e:
        lib.call("dirb200_gram_f64", C.c_void_p(x.data_ptr()), 2, 8068, C.c_void_p(mean.data_ptr()),
                 C.c_void_p(g.data_ptr()), ops._stream())
    assert e.value.status == -2                                          # DIRB200_ENOTSUP: above D = 8064
    with pytest.raises(lib.DirbError) as e:
        lib.call("dirb200_gram_f64", C.c_void_p(x.data_ptr()), 2, 6, C.c_void_p(mean.data_ptr()),
                 C.c_void_p(g.data_ptr()), ops._stream())
    assert e.value.status == -1                                          # DIRB200_EINVAL: D % 4 != 0 in the C ABI
    x8064 = torch.ones((3, 8064), dtype=torch.float32, device="cuda")
    m8064 = torch.ones(8064, dtype=torch.float64, device="cuda")
    assert float(ops.gram_f64(x8064, m8064).abs().max()) == 0.0           # the largest D runs (rows equal to the mean)


def _planted(n, d, seed=0):
    """Rows with a planted spectrum (geometric from 1 to 1e-4) on a random basis, mean ~0.1, fp32."""
    r = np.random.RandomState(seed)
    q, _ = np.linalg.qr(r.standard_normal((d, d)))
    lam = np.geomspace(1.0, 1e-4, d)
    z = r.standard_normal((n, d)).astype(np.float32) * np.sqrt(lam).astype(np.float32)
    return (z @ q.T.astype(np.float32) + 0.1 * r.uniform(-1, 1, d).astype(np.float32)).astype(np.float32)


def test_fit_matches_sklearn_and_whitens_alike():
    _gpu()
    from sklearn.decomposition import PCA
    from dirb200.whitening import fit_pca
    from dirtorch.utils import common
    n, d = 100000, 2048
    x = _planted(n, d)
    ours = fit_pca(torch.from_numpy(x).cuda())
    ref = PCA(whiten=True, svd_solver="full").fit(x.astype(np.float64))
    assert type(ours) is PCA and ours.n_components_ == d
    lam, lr = ours.explained_variance_, ref.explained_variance_
    ev_err = np.abs(lam - lr) / (1e-10 * lr + 1e-14 * lr[0])
    print("explained_variance_: max |d| / (1e-10 lambda + 1e-14 lambda_max) = %.3g" % ev_err.max())
    assert ev_err.max() <= 1.0
    np.testing.assert_allclose(ours.mean_, ref.mean_, rtol=0, atol=1e-12)
    gap = np.minimum(np.abs(np.diff(lr, prepend=np.inf)), np.abs(np.diff(lr, append=-np.inf)))
    sep = gap >= 1e-4 * lr[0]                         # components whose eigenvalue is separated from its neighbours
    comp_err = np.abs(ours.components_[sep] - ref.components_[sep]).max()
    print("components: %d gap-separated, max |d| %.3g" % (sep.sum(), comp_err))
    assert sep.sum() >= 100 and comp_err <= 1e-8
    xq = x[:2000]
    for p in (0.25, 0.5):
        for v in (None, 32):
            kw = dict(whitenp=p, whitenv=v, whitenm=2.0)
            err = rel_l2(common.whiten_features(xq, ours, **kw), common.whiten_features(xq, ref, **kw))
            print("whiten_features p=%g v=%s: ours vs sklearn's PCA rel L2 %.3g" % (p, v, err))
            assert err < 2e-5
    # sklearn's transform of our object = the project's transform (whitenp 0.5, whitenm 1 is sklearn's whitening)
    err = rel_l2(common.transform(ours, xq, whitenp=0.5), ours.transform(xq.astype(np.float64)))
    print("common.transform vs PCA.transform: rel L2 %.3g" % err)
    assert err < 2e-5


def test_fit_from_store_equals_fit_from_device(tmp_path):
    _gpu()
    from dirb200 import store as S
    from dirb200.whitening import fit_pca
    n, d = 30000, 132
    x = _planted(n, d, seed=4)
    st = S.write_store(str(tmp_path / "st"), x, rows_per_shard=7001)
    a = fit_pca(torch.from_numpy(x).cuda(), n_components=40)
    b = fit_pca(st, n_components=40, chunk_rows=4096)
    c = fit_pca(x, n_components=40, chunk_rows=10000)                    # host ndarray, streamed
    mean = x.astype(np.float64).sum(0) / n
    _, ga = M.gram_reference(x, mean)
    bound = M.gram_bound(n, ga) / (n - 1)
    for other in (b, c):
        np.testing.assert_allclose(other.mean_, a.mean_, rtol=0, atol=1e-12)
        assert np.all(np.abs(other.explained_variance_ - a.explained_variance_) <= 2 * bound.sum(0).max())
        assert np.abs(other.components_[:20] - a.components_[:20]).max() < 1e-8
    with pytest.raises(ValueError):
        bad = x.copy()
        bad[17, 3] = np.nan
        fit_pca(torch.from_numpy(bad).cuda())
    with pytest.raises(ValueError):
        bad[17, 3] = np.inf
        fit_pca(bad, chunk_rows=1000)


def test_learn_whiten_end_to_end(tmp_path, monkeypatch, capsys):
    """learn_whiten --dataset writes a checkpoint whose whitening gives test_dir the APs of the oracle pipeline with
    sklearn's PCA fit on the run's own saved descriptors."""
    _gpu()
    import e2e_data
    from sklearn.decomposition import PCA
    from oracle import dir_oracle as O
    root = str(tmp_path)
    gnd, names, qn, sd = e2e_data.build(root)
    ck = os.path.join(root, "ckpt.pt")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "model_options": dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3),
                "pca": {"Landmarks_clean": "kept as is"}}, ck)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    monkeypatch.setenv("DB_ROOT", root)
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", os.environ.get("CUDA_VISIBLE_DEVICES", "0"))
    from dirtorch import learn_whiten, test_dir
    out = os.path.join(root, "ckpt_w.pt")
    learn_whiten.learn_whiten_main(["--checkpoint", ck, "--name", "W", "--output", out, "--n-components", "32",
                                    "--dataset", 'ImageList("%s/list.txt", "%s/oxford5k/jpg")' % (root, root),
                                    "--threads", "2"])
    w = torch.load(out, map_location="cpu", weights_only=False)
    assert isinstance(w["pca"]["W"], PCA) and w["pca"]["Landmarks_clean"] == "kept as is"
    assert w["pca"]["W"].n_components_ == 32
    res = test_dir.test_dir_main(["--dataset", "Oxford5K", "--checkpoint", out, "--whiten", "W", "--whitenp", "0.25",
                                  "--gpu", "0", "--threads", "2", "--save-feats", os.path.join(root, "saved"),
                                  "--detailed"])
    saved = np.load(os.path.join(root, "saved", "feats.bdescs.npy"))
    ref_pca = PCA(n_components=32, whiten=True, svd_solver="full").fit(saved.astype(np.float64))
    W = O.whiten_features(saved, ref_pca, whitenp=0.25)
    ref_map, ref_aps = O.mean_ap(O.scores_exact(W[qn], W), gnd)
    np.testing.assert_allclose(res["APs"], ref_aps, rtol=0, atol=1e-12)
    assert abs(res["mAP"] - ref_map) < 1e-12
    # fitting again from the saved descriptors replaces the entry and says so
    out2 = os.path.join(root, "ckpt_w2.pt")
    learn_whiten.learn_whiten_main(["--checkpoint", out, "--name", "W", "--output", out2,
                                    "--load-feats", os.path.join(root, "saved", "feats.bdescs.npy")])
    assert "replacing the existing whitening 'W'" in capsys.readouterr().out
    w2 = torch.load(out2, map_location="cpu", weights_only=False)
    assert w2["pca"]["W"].n_components_ == min(len(names), 2048) and w2["pca"]["Landmarks_clean"] == "kept as is"
