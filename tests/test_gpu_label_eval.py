"""dirb200_index_count_ge on the GPU against the dense reference, and label-dataset evaluation through eval_model /
the test_dir command line against the literal dense-score path."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import label_model as LM  # noqa: E402
from oracle import dir_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _thresholds(q, db, r, max_thr):
    """Per query a random set of fp32 exact row scores (what positives give), descending."""
    s = O.scores_exact(q, db).astype(np.float32)
    off, thr = [0], []
    for i in range(q.shape[0]):
        k = r.randint(0, max_thr + 1)
        pick = r.randint(0, db.shape[0], k)
        thr.append(-np.sort(-s[i, pick]))
        off.append(off[-1] + k)
    return np.array(off, np.int64), np.concatenate(thr).astype(np.float32)


def _count(index, q, off, thr, skip=None):
    dev = torch.device("cuda")
    sk = None if skip is None else torch.from_numpy(np.asarray(skip, np.int64)).to(dev)
    c = index.count_ge(torch.from_numpy(q).to(dev), torch.from_numpy(off.astype(np.int32)).to(dev),
                       torch.from_numpy(thr).to(dev), sk)
    return c.cpu().numpy()


def _index(db, **kw):
    from dirb200 import ops
    return ops.Index(torch.from_numpy(db).cuda(), **kw)


@pytest.mark.parametrize("n,d,nq", [(1, 128, 7), (100, 128, 60), (100, 2048, 60), (30000, 128, 500), (30000, 2048, 200)])
def test_count_ge_bit_exact(n, d, nq):
    r = np.random.RandomState(n + d)
    db = _unit(r.standard_normal((n, d)))
    q = _unit(db[r.randint(0, n, nq)] + 0.7 * r.standard_normal((nq, d)).astype(np.float32))
    off, thr = _thresholds(q, db, r, 40)
    skip = r.randint(-1, n, nq)
    index = _index(db)
    np.testing.assert_array_equal(_count(index, q, off, thr, skip), LM.ge_counts(q, db, off, thr, skip))
    np.testing.assert_array_equal(_count(index, q, off, thr), LM.ge_counts(q, db, off, thr))


def test_count_ge_many_thresholds_exact_ties_non_unit():
    r = np.random.RandomState(11)
    n, d = 5000, 256
    db = _unit(r.standard_normal((n, d)))
    db[2500:2600] = db[:100]                                  # duplicated rows: identical scores, exact ties
    db *= r.uniform(0.3, 3.0, (n, 1)).astype(np.float32)      # non-unit rows (the eps bound scales with the norms)
    db[2500:2600] = db[:100]
    q = (_unit(r.standard_normal((3, d))) * np.float32(1.7)).astype(np.float32)
    s = O.scores_exact(q, db).astype(np.float32)
    thr0 = -np.sort(-s[0, r.choice(n, 2000, replace=False)])  # one query with 2000 thresholds
    thr1 = -np.sort(-s[1, np.r_[0:100, 2500:2600]])           # thresholds = scores of duplicated rows
    off = np.array([0, 2000, 2200, 2200], np.int64)
    thr = np.concatenate([thr0, thr1]).astype(np.float32)
    skip = np.array([5, 2510, -1])
    index = _index(db, check_norms=False)
    ref = LM.ge_counts(q, db, off, thr, skip)
    np.testing.assert_array_equal(_count(index, q, off, thr, skip), ref)
    # forced band everywhere, then forced band overflow -> exact recount: identical counts, the path shows in stats()
    index.set_option("count_eps", 1e-3)
    np.testing.assert_array_equal(_count(index, q, off, thr, skip), ref)
    assert index.stats()["candidates"] > 0
    index.set_option("band_cap", 16)
    np.testing.assert_array_equal(_count(index, q, off, thr, skip), ref)
    st = index.stats()
    assert st["retries"] >= 1 and st["candidates"] > 16
    with pytest.raises(Exception):
        _count(index, q, off, thr[::-1].copy(), skip)          # thresholds not descending: refused


def test_count_ge_sharded_sum():
    r = np.random.RandomState(4)
    n, d, nq = 3001, 128, 50
    db = _unit(r.standard_normal((n, d)))
    q = _unit(r.standard_normal((nq, d)))
    off, thr = _thresholds(q, db, r, 30)
    skip = r.randint(-1, n, nq)
    ref = _count(_index(db), q, off, thr, skip)
    np.testing.assert_array_equal(ref, LM.ge_counts(q, db, off, thr, skip))
    total = np.zeros_like(ref)
    for lo, hi in ((0, 700), (700, 700), (700, n)):             # uneven, one empty
        part = np.ascontiguousarray(db[lo:hi])
        total += _count(_index(part, index_offset=lo), q, off, thr, skip)
    np.testing.assert_array_equal(total, ref)


def _classes(r, n, d, lo, hi, sigma=0.6):
    sizes = []
    while sum(sizes) < n:
        sizes.append(int(r.randint(lo, hi + 1)))
    sizes[-1] -= sum(sizes) - n
    sizes = [s for s in sizes if s > 0]
    labels = np.repeat(np.arange(len(sizes)), sizes)
    r.shuffle(labels)
    centers = _unit(r.standard_normal((len(sizes), d)))
    x = _unit(centers[labels] + sigma * r.standard_normal((n, d)).astype(np.float32) / np.sqrt(d) * 8)
    return x, ["c%d" % v for v in labels]


def _same_res(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if k == "tops":
            assert a[k] == b[k]
        else:
            np.testing.assert_allclose(a[k], b[k], rtol=0, atol=1e-12)


def test_eval_model_label_datasets_match_dense(tmp_path):
    from dirtorch import datasets as D
    from dirb200.pipeline import eval_model
    r = np.random.RandomState(8)
    x, labels = _classes(r, 20000, 128, 1, 300)
    with open(tmp_path / "db.txt", "w") as f:
        f.write("\n".join("im%05d.jpg %s" % (i, l) for i, l in enumerate(labels)) + "\n")
    feats = tmp_path / "feats"
    os.makedirs(feats)
    np.save(feats / "feats.bdescs.npy", x)
    ds = D.ImageListLabels(str(tmp_path / "db.txt"), root=str(tmp_path))
    res = eval_model(ds, None, "", detailed=True, load_feats=str(feats))
    ref = eval_model(ds, None, "", detailed=True, load_feats=str(feats), dense_scores=True)
    _same_res(res, ref)
    assert 0 < res["mAP"] < 1 and len(res["APs"]) == 20000 and "top100" in res
    # separate query list, one label absent from the database
    qi = r.randint(0, 20000, 400)
    qlabels = [labels[i] for i in qi] + ["nowhere"]
    q = _unit(np.vstack([x[qi] + 0.02 * r.standard_normal((400, 128)).astype(np.float32), r.standard_normal((1, 128))]))
    with open(tmp_path / "q.txt", "w") as f:
        f.write("\n".join("q%05d.jpg %s" % (i, l) for i, l in enumerate(qlabels)) + "\n")
    np.save(feats / "feats.qdescs.npy", q)
    dsq = D.ImageListLabelsQ(str(tmp_path / "db.txt"), str(tmp_path / "q.txt"), root=str(tmp_path))
    res = eval_model(dsq, None, "", detailed=True, load_feats=str(feats))
    ref = eval_model(dsq, None, "", detailed=True, load_feats=str(feats), dense_scores=True)
    _same_res(res, ref)
    assert res["APs"][-1] == -1


def test_dir_main_on_label_list(tmp_path, monkeypatch):
    import synthdata as synth
    from dirtorch import test_dir
    r = np.random.RandomState(9)
    x, labels = _classes(r, 3000, 2048, 1, 60)
    with open(tmp_path / "db.txt", "w") as f:
        f.write("\n".join("im%05d.jpg %s" % (i, l) for i, l in enumerate(labels)) + "\n")
    feats = tmp_path / "feats"
    os.makedirs(feats)
    np.save(feats / "feats.bdescs.npy", x)
    sd = synth.make_state_dict("resnet50_rmac", seed=0)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()},
                "model_options": dict(arch="resnet50_rmac", out_dim=2048, pooling="gem", gemp=3)}, tmp_path / "ckpt.pt")
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", os.environ.get("CUDA_VISIBLE_DEVICES", "0"))
    args = ["--dataset", 'ImageListLabels("%s", root="%s")' % (tmp_path / "db.txt", tmp_path), "--checkpoint",
            str(tmp_path / "ckpt.pt"), "--whiten", "", "--gpu", "0", "--load-feats", str(feats), "--detailed"]
    _same_res(test_dir.test_dir_main(args), test_dir.test_dir_main(args + ["--dense-scores"]))
