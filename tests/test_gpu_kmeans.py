"""Spherical k-means on the GPU (DESIGN.md section 4.9, rules K1-K7).  -m gpu

A fit must equal tests/kmeans_model.py bit for bit: centres, labels, scores, iteration count and objective, for every
initialisation, with a planted empty cluster and a planted zero sum.  The relocation, update and k-means++ kernels are
also checked alone on inputs the fits do not reach (large clusters, ties in the scores, many empty clusters)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import kmeans_model as M  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mods():
    from dirb200 import cluster, lib, ops
    ops.require_gpu(0)
    return cluster, lib, ops


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _clustered(n, dim, k, seed=0, spread=0.35):
    r = np.random.RandomState(seed)
    c = _unit(r.standard_normal((k, dim)))
    return _unit(c[r.randint(0, k, n)] + spread * r.standard_normal((n, dim)) / np.sqrt(dim / 64))


def _bits(x):
    x = x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    return x.view(np.uint8)


def _gpu_scores(X, Cn):
    """The exact score matrix from Index.search(X, K) (every centre of every row, put back in centre order): the model's
    own restatement of exact_dot_warp is checked against it in test_model_scores_equal_the_search."""
    from dirb200 import ops
    idx = ops.Index(_t(Cn), check_norms=False)
    try:
        s, i = idx.search(_t(X), Cn.shape[0])
    finally:
        idx.close()
    E = np.empty((X.shape[0], Cn.shape[0]))
    np.put_along_axis(E, i.cpu().numpy(), s.cpu().numpy(), axis=1)
    return E


def _fit(X, k, **kw):
    return M.fit(X, k, scores=_gpu_scores, **kw)


def _same_fit(km, ref):
    assert km.n_iter_ == ref["n_iter"]
    assert np.array_equal(km.labels_.cpu().numpy(), ref["labels"])
    assert np.array_equal(_bits(km.scores_), _bits(ref["scores"]))
    assert np.array_equal(_bits(km.cluster_centers_), _bits(ref["centres"]))
    assert km.objective_ == ref["objective"]
    assert (km.stats_["relocations"], km.stats_["zero_sums"]) == (ref["relocations"], ref["zero_sums"])


# ------------------------------------------------------------------------------------------------ Index.nearest (K2 / K3)
def _check_nearest(X, Cn, **opts):
    _, _, ops = _mods()
    idx = ops.Index(_t(Cn), check_norms=False)
    try:
        for key, v in opts.items():
            idx.set_option(key, v)
        q = _t(X)
        lab, sc = idx.nearest(q)
        st = idx.nearest_stats()
        s1, i1 = idx.search(q, 1)
    finally:
        idx.close()
    assert np.array_equal(lab.cpu().numpy(), i1[:, 0].cpu().numpy())
    assert np.array_equal(_bits(sc), _bits(s1[:, 0]))
    return st


@pytest.mark.parametrize("n,dim,k", [(5000, 64, 1), (5000, 64, 31), (5000, 64, 32), (5000, 64, 33), (20000, 2048, 128),
                                     (20000, 2048, 129), (200000, 64, 4096), (30000, 2048, 65536)])
def test_nearest_equals_search_top1(n, dim, k):
    r = np.random.RandomState(k)
    X = _clustered(max(n, k), dim, max(2, k // 4), seed=k)
    Cn = X[r.permutation(len(X))[:k]].copy()                   # centres that are rows
    if k > 2:
        Cn[k // 2] = Cn[0]                                     # a duplicated centre: the smaller index wins
        Cn[-1] = Cn[1]
    st = _check_nearest(X[:n], Cn)
    assert st["full_rescores"] <= st["band_rows"] <= n and st["rescored"] >= n


def test_nearest_all_rows_and_small_workspace():
    X = _clustered(3000, 256, 40, seed=3)
    Cn = np.repeat(X[:1], 70, axis=0)                          # all-equal centres: every group ties
    st = _check_nearest(X, Cn)
    assert st["band_rows"] == 3000
    st = _check_nearest(X, X[:500], nearest_cap=0)             # every row re-scored over all centres
    assert st["full_rescores"] == 3000 and st["rescored"] == 3000 * 500
    _check_nearest(X, X[:500], ws_budget=1)                    # blocks of 128 queries


def test_assign_on_both_sides_of_the_nearest_limit():
    cluster, _, ops = _mods()
    X = _clustered(4000, 64, 50, seed=12)
    for k in (cluster.NEAREST_MAX_K, cluster.NEAREST_MAX_K + 1):
        Cn = _clustered(k, 64, 50, seed=13)
        lab, sc = cluster.assign(_t(X), _t(Cn))
        idx = ops.Index(_t(Cn), check_norms=False)
        s1, i1 = idx.search(_t(X), 1)
        idx.close()
        assert np.array_equal(lab.cpu().numpy(), i1[:, 0].cpu().numpy()) and np.array_equal(_bits(sc), _bits(s1[:, 0]))


# ------------------------------------------------------------------------------------------------ fits against the model
@pytest.mark.parametrize("n,dim,k", [(3000, 64, 33), (1000, 2048, 129)])
def test_model_scores_equal_the_search(n, dim, k):
    _mods()
    X = _clustered(n, dim, 20, seed=k)
    E = _gpu_scores(X, X[:k])
    assert np.array_equal(_bits(E), _bits(M.exact_scores(X, X[:k])))


@pytest.mark.parametrize("init", ["k-means++", "random", "array"])
def test_fit_equals_model(init):
    cluster, _, _ = _mods()
    X = _clustered(20000, 256, 100, seed=1)
    arg = _unit(np.random.RandomState(2).standard_normal((100, 256))) if init == "array" else init
    ref = _fit(X, 100, init=arg, max_iter=20, seed=5)
    km = cluster.SphericalKMeans(100, init=arg, max_iter=20, seed=5).fit(_t(X))
    _same_fit(km, ref)
    again = cluster.SphericalKMeans(100, init=arg, max_iter=20, seed=5).fit(X)      # host input, second run
    for a, b in ((km.cluster_centers_, again.cluster_centers_), (km.labels_, again.labels_), (km.scores_, again.scores_)):
        assert np.array_equal(_bits(a), _bits(b))
    assert np.array_equal(km.predict(_t(X)).cpu().numpy(), km.labels_.cpu().numpy())


def test_planted_empty_cluster():
    cluster, _, _ = _mods()
    r = np.random.RandomState(3)
    centres = _unit(r.standard_normal((8, 256)))
    truth = r.randint(0, 8, 3000)
    X = _unit(centres[truth] + 0.02 * r.standard_normal((3000, 256)))
    first = [int(np.nonzero(truth == c)[0][0]) for c in range(8)]
    init = np.concatenate([X[first], -X[first[:2]]])        # clusters 8 and 9 are nobody's nearest
    ref = _fit(X, 10, init=init, max_iter=20)
    km = cluster.SphericalKMeans(10, init=init).fit(_t(X))
    _same_fit(km, ref)
    assert ref["relocations"] >= 2


def test_planted_zero_sum():
    """Cluster 0 is {x, -x}: x is orthogonal to every centre (all scores 0, so both go to the smallest centre), and no
    other row is nearest to centre 0."""
    cluster, _, _ = _mods()
    r = np.random.RandomState(4)
    X = np.abs(r.standard_normal((2000, 256))).astype(np.float32)
    X[:, 128:] = 0
    X = _unit(X)
    X[100] = 0
    X[100, 200] = 1
    X[1500] = -X[100]
    init = np.zeros((6, 256), np.float32)
    init[0, :128] = -1 / np.sqrt(np.float32(128))
    init[1:] = X[:5]                                           # every other centre starts on a row of its own
    ref = _fit(X, 6, init=init, max_iter=20)
    assert ref["zero_sums"] >= 1 and ref["labels"][100] == ref["labels"][1500] == 0
    km = cluster.SphericalKMeans(6, init=init).fit(_t(X))
    _same_fit(km, ref)


def test_max_iter_and_small_cases():
    cluster, _, _ = _mods()
    X = _clustered(1500, 64, 20, seed=6)
    for k, init, it in ((1, "k-means++", 20), (31, "random", 1), (32, "k-means++", 0), (33, "random", 3),
                        (1500, "random", 2)):
        ref = _fit(X, k, init=init, max_iter=it, seed=k)
        km = cluster.SphericalKMeans(k, init=init, max_iter=it, seed=k).fit(_t(X))
        _same_fit(km, ref)


# ------------------------------------------------------------------------------------------------ kernels alone
def test_update_kernel_with_large_clusters():
    _, lib, ops = _mods()
    r = np.random.RandomState(7)
    X = _unit(r.standard_normal((6000, 2048)))
    labels = np.where(r.rand(6000) < 0.9, 1, r.randint(0, 4, 6000)).astype(np.int64)     # cluster 1: ~5 500 rows
    labels[labels == 3] = 2                                                             # cluster 3 empty
    C0 = _unit(r.standard_normal((4, 2048)))
    ref, zero = M.update(X, labels, C0)
    x, lab, cen = _t(X), _t(labels), _t(C0.copy())
    ws = torch.empty(lib.raw("dirb200_kmeans_update_workspace_bytes")(6000, 4, 2048), dtype=torch.uint8, device=DEV)
    z = C.c_int64()
    counts = _t(np.bincount(labels, minlength=4).astype(np.int32))
    lib.call("dirb200_kmeans_update", ops._ptr(x), 6000, 2048, ops._ptr(lab), ops._ptr(counts), 4, ops._ptr(cen), ops._ptr(ws),
             C.byref(z), ops._stream())
    assert z.value == zero == 1
    assert np.array_equal(_bits(cen), _bits(ref))


def test_relocation_kernel_with_ties_and_many_empty_clusters():
    _, lib, ops = _mods()
    r = np.random.RandomState(8)
    n, k = 50000, 3000
    labels = r.randint(0, 1000, n).astype(np.int64)              # clusters 1000 .. 2999 empty
    labels[:5] = 1000 + np.arange(5)                             # a few singletons among them
    scores = np.round(r.uniform(-1, 1, n), 2)                    # many ties: the row decides
    want, moves = M.relocate(labels, scores, k)
    lab, sc = _t(labels), _t(scores)
    counts = torch.empty(k, dtype=torch.int32, device=DEV)
    ws = torch.empty(256, dtype=torch.uint8, device=DEV)
    out = (C.c_int64 * 3)()
    lib.call("dirb200_kmeans_stats", ops._ptr(lab), ops._ptr(sc), None, n, k, ops._ptr(ws), ops._ptr(counts), out, ops._stream())
    assert out[0] == n and out[1] == M.objective_units(scores) and out[2] == k - 1005
    ws = torch.empty(lib.raw("dirb200_kmeans_relocate_workspace_bytes")(n), dtype=torch.uint8, device=DEV)
    mv = C.c_int64()
    lib.call("dirb200_kmeans_relocate", ops._ptr(lab), ops._ptr(sc), n, k, ops._ptr(counts), ops._ptr(ws), C.byref(mv),
             ops._stream())
    assert mv.value == moves == k - 1005
    assert np.array_equal(lab.cpu().numpy(), want)
    assert np.array_equal(counts.cpu().numpy(), np.bincount(want, minlength=k))


def test_kmeans_pp_kernel():
    cluster, _, _ = _mods()
    X = _clustered(300000, 64, 50, seed=9)                    # 1172 weight blocks: the block search crosses a chunk
    assert np.array_equal(cluster.kmeans_pp_rows(_t(X), 20, 11), M.kmeans_pp(X, 20, 11))
    basis = np.repeat(np.eye(64, dtype=np.float32)[:3], 10, axis=0)
    with pytest.raises(ValueError):
        cluster.kmeans_pp_rows(_t(basis), 4, 0)


# ------------------------------------------------------------------------------------------------ errors
def test_errors():
    cluster, _, _ = _mods()
    X = _clustered(100, 64, 4)
    bad = X.copy()
    bad[3] *= 1.01
    K = cluster.SphericalKMeans
    for km, data in ((K(4), bad), (K(0), X), (K(101), X), (K(4, init="kmeans"), X), (K(4, init=X[:3]), X),
                     (K(4, init=X[:4, :32].copy()), X), (K(4, max_iter=-1), X), (K(2.5), X),
                     (K(4), _unit(np.random.RandomState(0).standard_normal((100, 96))))):
        with pytest.raises(ValueError):
            km.fit(_t(data))
    km = K(4).fit(_t(X))
    with pytest.raises(ValueError):
        km.predict(_t(np.zeros((3, 128), np.float32)))
    with pytest.raises(ValueError):
        K(4).predict(_t(X))


# ------------------------------------------------------------------------------------------------ command line
def test_cluster_features_end_to_end(tmp_path, monkeypatch, capsys):
    import json
    import e2e_data
    root = str(tmp_path)
    _, names, _, sd = e2e_data.build(root)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "model_options": dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)},
               os.path.join(root, "ckpt.pt"))
    monkeypatch.setenv("DB_ROOT", root)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    dataset = 'ImageList("%s/list.txt", "%s/oxford5k/jpg")' % (root, root)
    from dirtorch import cluster_features, extract_features
    feats_npy = os.path.join(root, "feats.npy")
    extract_features.extract_features_main(["--dataset", dataset, "--checkpoint", os.path.join(root, "ckpt.pt"),
                                            "--output", feats_npy, "--gpu", "0", "--threads", "2"])
    F = np.load(feats_npy)
    ref = _fit(F, 8, init="random", max_iter=20, seed=2)
    out = os.path.join(root, "km.npz")
    js = os.path.join(root, "km.json")
    res = cluster_features.cluster_features_main(["--load-feats", feats_npy, "--n-clusters", "8", "--init", "random",
                                                  "--seed", "2", "--output", out, "--out-json", js])
    assert np.array_equal(res["labels"], ref["labels"])
    z = np.load(out)
    assert set(z.files) == {"labels", "scores", "centres"} and np.array_equal(_bits(z["centres"]), _bits(ref["centres"]))
    rows = json.load(open(js))["clusters"]
    assert rows == [np.nonzero(ref["labels"] == c)[0].tolist() for c in range(8)]
    assert "%d rows in 8 clusters" % len(F) in capsys.readouterr().out
    res2 = cluster_features.cluster_features_main(["--dataset", dataset, "--checkpoint", os.path.join(root, "ckpt.pt"),
                                                   "--n-clusters", "8", "--init", "random", "--seed", "2", "--out-json",
                                                   js, "--threads", "2"])
    assert np.array_equal(res2["labels"], ref["labels"])
    assert json.load(open(js))["clusters"] == [[names[i] for i in np.nonzero(ref["labels"] == c)[0]] for c in range(8)]
