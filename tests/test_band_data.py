"""The band-edge constructions of tests/band_data.py, checked on the CPU: grid exactness, the planted fp16-path gaps,
that the search protocol model needs its full band on them, and the hand-derived label counts at rounding midpoints."""
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import band_data as B  # noqa: E402
import label_model as LM  # noqa: E402
import search_model as M  # noqa: E402
from oracle import dir_oracle as O  # noqa: E402


def _fraction_dot(q, r):
    return sum((Fraction(float(a)) * Fraction(float(b)) for a, b in zip(q, r) if a and b), Fraction(0))


@pytest.mark.parametrize("mag", [2.0 ** -3, 2.0 ** -6, 0.7, 3e-5, 2.0 ** -20, 17.0])
def test_near_midpoint_rounds_the_stated_way(mag):
    for up in (False, True):
        v = np.float32(B.near_midpoint(mag, up))
        assert float(v) == B.near_midpoint(mag, up)                      # representable in fp32
        h = float(np.float16(v))
        sp = B.f16_spacing(mag)
        assert abs(h - float(v)) >= sp / 2 * (1 - 2.0 ** -8)              # half a spacing, nearly
        assert (h > float(v)) == up


@pytest.mark.parametrize("D", [64, 256, 1024, 2048])
def test_probe_families_sit_on_the_bound_and_score_exactly(D):
    for name, (q, rows) in B.probe_families(D).items():
        assert np.linalg.norm(q.astype(np.float64)) <= 1.0 and np.linalg.norm(rows.astype(np.float64), axis=1).max() <= 1.0
        ex = M.exact_scores(q[None], rows)[0]
        assert np.array_equal(ex, O.scores_exact(q[None], rows)[0])       # any summation order gives the same bits
        assert all(Fraction(float(e)) == _fraction_dot(q, r) for e, r in zip(ex, rows))
        err = M.fast_scores(q[None], rows)[0].astype(np.float64) - ex
        assert np.abs(err).max() <= B.EPS16
        assert np.abs(err).min() > 9.0e-4 if D >= 256 else np.abs(err).min() > 8.5e-4, (name, err)
        if name == "decoy_trap":
            assert (err[:2] > 0).all() and (err[2:] < 0).all()
            assert ex[2:].min() > ex[:2].max()                              # traps outrank decoys exactly


@pytest.mark.parametrize("D", [64, 256, 1024, 2048])
def test_planted_gap_lies_between_the_reduced_and_the_full_band(D):
    db, q, info = B.topk_layout(D, 1200, n_dec=16, n_trap=8, seed=D)
    fast = M.fast_scores(q[None], db)[0]
    ex = M.exact_scores(q[None], db)[0]
    dec, trp = info["decoy"], info["trap"]
    assert ex[trp].min() >= B.MU and ex[dec].max() <= 0
    gap_min = fast[dec].min() - fast[trp].max()
    gap_max = fast[dec].max() - fast[trp].min()
    assert 1.5e-3 < gap_min <= gap_max < 2 * B.EPS16 - 3e-4, (gap_min, gap_max)
    rest = np.setdiff1d(np.arange(db.shape[0]), np.concatenate([dec, trp]))
    assert ex[rest].max() < ex[dec].min() - 5e-3 and fast[rest].max() < fast[trp].min() - 5e-3
    assert np.abs(fast - ex).max() <= B.EPS16


def _model_exact(db, q, k, bounds, monkeypatch, band, **kw):
    monkeypatch.setattr(M, "BAND", np.float32(band))
    got_s, got_i, _ = M.sharded_search(q[None], db, k, bounds, **kw)
    ref_s, ref_i = M.exact_topk(q[None], db, k)
    return np.array_equal(got_i, ref_i) and np.array_equal(got_s, ref_s)


@pytest.mark.parametrize("layout", ["dense", "filter", "retry", "two_shards"])
def test_search_model_needs_the_full_band_on_decoys_and_traps(layout, monkeypatch):
    """search_model at its BAND = 2 eps16 returns the exact top-k; at 1.25 eps16 it misses the traps."""
    D = 256
    if layout == "two_shards":
        db, q, bounds, info = B.two_shard_layout(D, 1500, 1500)
        kw = {"sample_rows": 8192}
    else:
        db, q, info = B.topk_layout(D, 3000, n_mid=300 if layout == "retry" else 0, seed_groups=layout != "retry")
        bounds = [(0, db.shape[0])]
        kw = {"dense": {"sample_rows": 8192}, "filter": {"sample_rows": 512},
              "retry": {"sample_rows": 256, "cand_cap": 256}}[layout]
    k = info["k"]
    ref_s, ref_i = M.exact_topk(q[None], db, k)
    assert set(info["trap"]) <= set(ref_i[0])
    assert _model_exact(db, q, k, bounds, monkeypatch, 2 * B.EPS16, **kw)
    assert not _model_exact(db, q, k, bounds, monkeypatch, 1.25 * B.EPS16, **kw)


def test_rank_layout_counts():
    db, q, info = B.rank_layout(256, 2000)
    t = info["target"]
    _, above = O.rank_counts(q[None], db, [0, 1], [t])
    assert above[0] == len(info["strong"]) + len(info["trap"])              # derived by hand
    fast = M.fast_scores(q[None], db)[0]
    ex = M.exact_scores(q[None], db)[0]
    s = ex[t]
    assert (ex[info["decoy"]] < s).all() and (ex[info["trap"]] > s).all()
    assert (fast[info["decoy"]] - s > 9e-4).all() and (s - fast[info["trap"]] > 9e-4).all()
    assert (np.abs(fast[info["decoy"]] - s) < B.EPS16).all() and (np.abs(s - fast[info["trap"]]) < B.EPS16).all()


@pytest.mark.parametrize("scale", [2.0 ** -10, 2.0 ** 7])
def test_unnormalised_recipe_on_the_model(scale, monkeypatch):
    """Rows of norm ~1e-3 have subnormal fp16 entries: 1.2e-3 |q| |row| is too small a bound there, the corrected
    recipe (band_data.unnormalised_eps16) holds; rows of norm ~100 are covered by either."""
    D = 2048
    db, q, info = B.topk_layout(D, 1200, scale=scale)
    qn = float(np.linalg.norm(q.astype(np.float64)))
    rn = float(np.linalg.norm(db.astype(np.float64), axis=1).max())
    ex = M.exact_scores(q[None], db)[0]
    fast = M.fast_scores(q[None], db)[0].astype(np.float64)
    old, new = 1.2e-3 * qn * rn, B.unnormalised_eps16(qn, rn, D)
    assert np.abs(fast - ex).max() <= new
    bounds, kw = [(0, db.shape[0])], {"sample_rows": 8192}
    assert _model_exact(db, q, info["k"], bounds, monkeypatch, 2 * new, **kw)
    if scale < 1:
        assert np.abs(db[info["decoy"], :-2]).max() < 2.0 ** -14                # subnormal in fp16
        assert np.abs(fast - ex).max() > old
        assert not _model_exact(db, q, info["k"], bounds, monkeypatch, 2 * old, **kw)
    else:
        assert _model_exact(db, q, info["k"], bounds, monkeypatch, 2 * old, **kw)


def test_midpoint_rows_are_exact_in_any_order_and_cover_the_edges():
    q, db, exact, thr = B.midpoint_data()
    for r, e in zip(db, exact):
        assert Fraction(e) == _fraction_dot(q, r)
    assert np.array_equal(O.scores_exact(q[None], db)[0], exact)
    evens = [LM.even_significand(s) for s in thr if s != 0]
    assert any(evens) and not all(evens)
    assert any(s < 0 for s in thr) and 0.0 in thr.tolist()
    assert {float(s) for s in thr} >= {0.5, 2.0 ** -10, -0.25, 1.0, -1.0}   # binade edges
    assert np.signbit(thr).sum() > (thr < 0).sum()                          # -0 is there


def test_midpoint_counts_by_hand_equal_label_model():
    q, db, exact, thr = B.midpoint_data()
    i = 0
    for s in thr:                                                          # the rule, row by row
        for label, _, e in B.midpoint_rows(s):
            reach = np.float32(e) >= s
            want = {"s": True, "pred": False, "m-": False, "m+": True, "m": LM.even_significand(s)}[label]
            assert reach == want, (s, label)
            assert float(exact[i]) == e or (e == 0 and exact[i] == 0)
            i += 1
    off = np.array([0, thr.shape[0]])
    hand = B.ge_counts_by_hand(exact, thr)
    assert np.array_equal(LM.ge_counts(q[None], db, off, thr), hand)
    assert np.array_equal(LM.ge_counts(q[None], db, off, thr, skip=[7]), B.ge_counts_by_hand(exact, thr, skip=7))
