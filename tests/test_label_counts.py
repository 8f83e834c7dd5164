"""Host side of label AP from threshold counts (dirb200_index_count_ge): the AP formula, top-k from a ranking, the
positives' CSR, and the rounding-boundary rule of the kernel's epilogue."""
import os
import sys

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st
from sklearn.metrics import average_precision_score

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import label_model as LM  # noqa: E402


def _write(path, names, labels):
    with open(path, "w") as f:
        f.write("\n".join("%s %s" % (n, l) for n, l in zip(names, labels)) + "\n")


def _labelled(tmp_path, labels, qlabels=None):
    from dirtorch import datasets as D
    _write(tmp_path / "db.txt", ["im%04d.jpg" % i for i in range(len(labels))], labels)
    if qlabels is None:
        return D.ImageListLabels(str(tmp_path / "db.txt"), root=str(tmp_path))
    _write(tmp_path / "q.txt", ["q%04d.jpg" % i for i in range(len(qlabels))], qlabels)
    return D.ImageListLabelsQ(str(tmp_path / "db.txt"), str(tmp_path / "q.txt"), root=str(tmp_path))


def _aps_from_rows(ds, scores):
    """What the GPU path computes, from a dense fp32 score matrix: thresholds = the positives' scores (descending),
    counts = rows (the skip row excluded) at or above each."""
    off, rows, skip = ds.label_targets()
    aps = []
    for q in range(len(off) - 1):
        row = np.asarray(scores[q], dtype=np.float32)
        thr = -np.sort(-row[rows[off[q]:off[q + 1]]])
        keep = np.ones(row.shape[0], bool)
        if skip[q] >= 0:
            keep[skip[q]] = False
        cnt = (row[keep][None, :] >= thr[:, None]).sum(1)
        aps.append(ds.eval_query_AP_from_ge_counts(q, thr, cnt))
    return np.array(aps, dtype=np.float64)


@pytest.mark.parametrize("separate_queries", [False, True])
def test_ap_from_ge_counts_equals_sklearn_with_ties(tmp_path, separate_queries):
    r = np.random.RandomState(3)
    n = 300
    labels = ["c%d" % v for v in r.randint(0, 12, n)]
    labels[7] = "alone"
    qlabels = ["c%d" % v for v in r.randint(0, 14, 40)] + ["alone", "nowhere"] if separate_queries else None
    ds = _labelled(tmp_path, labels, qlabels)
    nq = len(qlabels) if separate_queries else n
    scores = np.round(r.standard_normal((nq, n)) * 4).astype(np.float32) / 8    # few distinct values: many exact ties
    aps = _aps_from_rows(ds, scores)
    ref = np.array([ds.eval_query_AP(q, scores[q]) for q in range(nq)], dtype=np.float64)
    np.testing.assert_allclose(aps, ref, rtol=0, atol=1e-12)
    # and directly against sklearn on the kept entries of the dense row
    for q in range(nq):
        gt = ds.get_query_groundtruth(q)
        keep = gt != 0
        if (gt[keep] > 0).any():
            assert abs(aps[q] - average_precision_score(gt[keep] > 0, scores[q][keep])) < 1e-12
        else:
            assert aps[q] == -1
    if separate_queries:
        assert aps[-1] == -1 and aps[-2] >= 0                 # label absent from the database / class of one row
    else:
        assert aps[7] == -1


def test_ap_from_ge_counts_matches_reference_golden(golden, tmp_path):
    g = golden("label_ap.npz")
    labels, qlabels = [str(v) for v in g["labels"]], [str(v) for v in g["qlabels"]]
    ds = _labelled(tmp_path, labels)
    np.testing.assert_allclose(_aps_from_rows(ds, g["scores"]), g["aps"], rtol=0, atol=1e-12)
    dsq = _labelled(tmp_path, labels, qlabels)
    qaps = _aps_from_rows(dsq, g["qscores"])
    ok = np.isfinite(g["qaps"])
    np.testing.assert_allclose(qaps[ok], g["qaps"][ok], rtol=0, atol=1e-12)
    assert (qaps[~ok] == -1).all()


def test_label_targets_csr(tmp_path):
    labels = ["a", "b", "a", "c", "a", "b"]
    ds = _labelled(tmp_path, labels)
    off, rows, skip = ds.label_targets()
    assert off.tolist() == [0, 2, 3, 5, 5, 7, 8]
    assert [rows[off[q]:off[q + 1]].tolist() for q in range(6)] == [[2, 4], [5], [0, 4], [], [0, 2], [1]]
    assert skip.tolist() == list(range(6))
    off2, rows2, skip2 = ds.label_targets([4, 1])
    assert off2.tolist() == [0, 2, 3] and rows2.tolist() == [0, 2, 5] and skip2.tolist() == [4, 1]
    dsq = _labelled(tmp_path, labels, ["b", "z", "a"])
    off, rows, skip = dsq.label_targets()
    assert off.tolist() == [0, 2, 2, 5] and rows.tolist() == [1, 5, 0, 2, 4] and skip.tolist() == [-1, -1, -1]


def test_top_from_ranking_equals_eval_query_top(tmp_path):
    r = np.random.RandomState(5)
    n = 250
    labels = ["c%d" % v for v in r.randint(0, 30, n)]
    for qlabels in (None, ["c%d" % v for v in r.randint(0, 33, 20)]):
        ds = _labelled(tmp_path, labels, qlabels)
        nq = n if qlabels is None else len(qlabels)
        scores = r.permutation(nq * n).reshape(nq, n).astype(np.float32)     # distinct: no tie straddles any k
        for q in range(nq):
            ranked = np.argsort(-scores[q], kind="stable")[:100]
            assert ds.eval_query_top_from_ranking(q, ranked) == ds.eval_query_top(q, scores[q])
    small = _labelled(tmp_path, labels[:7])
    s = np.arange(7, dtype=np.float32)[::-1].copy()
    assert small.eval_query_top_from_ranking(0, np.arange(7)) == small.eval_query_top(0, s)


# ---- the epilogue's decision rule: decided (reached / not reached) or band, against brute-force fl32(e) >= s
# (scores are dot products of finite rows: the fp32 overflow boundary is out of scope)
_F32 = st.floats(width=32, min_value=-(2.0 ** 126), max_value=2.0 ** 126)
_SPECIAL = st.sampled_from([0.0, -0.0, 1.0, -1.0, 0.5, 2.0, 0.25, 1e-45, -1e-45, 1.1754944e-38, 2.0 ** 126])


def _reaches(e, s):
    return bool(np.float32(e) >= np.float32(s))


def _exact_rule(e, s):
    m = LM.boundary(s)
    return e > m or (e == m and LM.even_significand(s))


@settings(max_examples=3000, deadline=None)
@given(s=st.one_of(_F32, _SPECIAL), step=st.integers(-3, 3), eps_ulps=st.integers(0, 4), off=st.integers(-4, 4))
def test_decision_rule_reproduces_fp32_rounding(s, step, eps_ulps, off):
    s = np.float32(s)
    m = LM.boundary(s)
    # e on the boundary, or a few fp64 ulps either side of it
    e = m
    for _ in range(abs(step)):
        e = float(np.nextafter(e, np.inf if step > 0 else -np.inf))
    assert _exact_rule(e, s) == _reaches(e, s)
    # the tensor-core score x lies within eps of e; a decided answer must be the brute-force one
    eps = eps_ulps * float(np.spacing(abs(e) if e != 0 else 5e-324))
    x = e
    for _ in range(min(abs(off), eps_ulps)):
        x = float(np.nextafter(x, np.inf if off > 0 else -np.inf))
    if abs(x - e) > eps:                  # (steps of x across a binade boundary can exceed e's ulps)
        return
    d = LM.decide(x, eps, s)
    assert d is None or d == _reaches(e, s)
    if eps == 0 and x == e and e != m:
        assert d == _reaches(e, s)


@settings(max_examples=2000, deadline=None)
@given(s=_F32, e=st.floats(allow_nan=False, allow_infinity=False, min_value=-1e30, max_value=1e30))
def test_decision_rule_random_scores(s, e):
    assert _exact_rule(e, np.float32(s)) == _reaches(e, s)
    d = LM.decide(e, 0.0, s)
    assert d is None or d == _reaches(e, s)


def test_binade_and_zero_boundaries():
    for s in (1.0, 2.0, 0.5, -1.0, -2.0, 0.0, -0.0, np.float32(2.0 ** -126)):
        s = np.float32(s)
        m = LM.boundary(s)
        for e in (m, np.nextafter(m, np.inf), np.nextafter(m, -np.inf)):
            assert _exact_rule(float(e), s) == _reaches(float(e), s), (s, e)
    assert _reaches(LM.boundary(np.float32(0.0)), 0.0)          # -2^-150 rounds to -0, which is >= +0
