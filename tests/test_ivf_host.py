"""Inverted-file search on the CPU (DESIGN.md section 4.10): the model of tests/ivf_model.py against dense restatements
of rules I2-I5 and I7, a mirror of the device tile-table builder, six planted bugs, and spills of the new kernels."""
import os
import re

import numpy as np
import pytest

import ivf_model as M
import kmeans_model as KM
from conftest import REPO
from search_model import BAND, fast_scores


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _case(seed, n=400, d=64, k=9, nq=12, ties=True):
    r = np.random.RandomState(seed)
    C = _unit(r.standard_normal((k, d)))
    X = _unit(C[r.randint(0, k, n)] + 0.3 * r.standard_normal((n, d)) / 8)
    if ties:
        X[5] = X[3]                     # equal scores: ties go to the smaller row
        C[k - 1] = C[0]                 # a duplicated centre: probe ties, an empty list
    q = _unit(C[r.randint(0, k, nq)] + 0.3 * r.standard_normal((nq, d)) / 8)
    E, Ec = KM.exact_scores(q, X), KM.exact_scores(q, C)
    labels = KM.assign(KM.exact_scores(X, C))[0]
    return X, C, q, E, Ec, labels


def _dense_search(E, Ec, labels, nprobe, k):
    """I3 / I4 restated: sort centres by (-e, c), keep the rows whose label is among the first nprobe, sort them by
    (-e, row)."""
    out_s = np.full((E.shape[0], k), -np.inf)
    out_i = np.full((E.shape[0], k), -1)
    for q in range(E.shape[0]):
        P = sorted(range(Ec.shape[1]), key=lambda c: (-Ec[q, c], c))[:nprobe]
        rows = sorted((r for r in range(E.shape[1]) if labels[r] in P), key=lambda r: (-E[q, r], r))[:k]
        out_s[q, :len(rows)] = E[q, rows]
        out_i[q, :len(rows)] = rows
    return out_s, out_i


@pytest.mark.parametrize("seed", range(4))
def test_model_equals_dense_restatement(seed):
    X, C, q, E, Ec, labels = _case(seed)
    perm, off = M.build(labels, C.shape[0])
    assert off[-1] - off[-2] == 0                      # the duplicated centre's list is empty
    for nprobe in (1, 2, C.shape[0]):
        for k in (1, 7, 500):
            s, i = M.search(E, M.probe(Ec, nprobe), perm, off, k)
            ds, di = _dense_search(E, Ec, labels, nprobe, k)
            assert np.array_equal(i, di) and np.array_equal(s, ds)
    # every list probed: the exact top-k of all rows
    s, i = M.search(E, M.probe(Ec, C.shape[0]), perm, off, 50)
    assert np.array_equal(i, np.lexsort((np.broadcast_to(np.arange(X.shape[0]), E.shape), -E))[:, :50])


def test_band_keeps_every_row_of_the_exact_top_k():
    for seed in range(4):
        X, C, q, E, Ec, labels = _case(seed, n=600)
        perm, off = M.build(labels, C.shape[0])
        F = fast_scores(q, X)
        for nprobe in (1, 3):
            probes = M.probe(Ec, nprobe)
            for k in (1, 10, 40):
                top = M.search(E, probes, perm, off, k)[1]
                cand = M.candidates(F, probes, perm, off, k, BAND)
                for qi in range(q.shape[0]):
                    assert set(top[qi][top[qi] >= 0]) <= set(cand[qi])
                    assert set(cand[qi]) <= set(M.union(probes[qi], perm, off))


def test_rank_model_equals_dense_restatement():
    X, C, q, E, Ec, labels = _case(7)
    perm, off = M.build(labels, C.shape[0])
    r = np.random.RandomState(0)
    t_q = np.repeat(np.arange(q.shape[0]), 5)
    t_rows = r.randint(0, X.shape[0], t_q.shape[0])
    for nprobe in (1, 3, C.shape[0]):
        probes = M.probe(Ec, nprobe)
        got = M.ranks(E, probes, perm, off, t_q, t_rows)
        for i, (qi, t) in enumerate(zip(t_q, t_rows)):
            R = set(M.union(probes[qi], perm, off))
            L = sorted(R, key=lambda x: (-E[qi, x], x)) + sorted(set(range(X.shape[0])) - R, key=lambda x: (-E[qi, x], x))
            assert got[i] == L.index(t)
        if nprobe == C.shape[0]:
            assert np.array_equal(got, [int(((E[a] > E[a, t]) | ((E[a] == E[a, t]) & (np.arange(X.shape[0]) < t))).sum())
                                        for a, t in zip(t_q, t_rows)])


def _table_case(seed, sizes):
    r = np.random.RandomState(seed)
    K = len(sizes)
    labels = np.repeat(np.arange(K), sizes)
    r.shuffle(labels)
    perm, off = M.build(labels, K)
    Q = int(r.randint(1, 300))
    nprobe = int(r.randint(1, K + 1))
    probes = np.stack([r.permutation(K)[:nprobe] for _ in range(Q)])
    return perm, off, probes


SIZES = [[0, 1, 127, 128, 129, 0, 300], [500], [0, 0, 500, 0], [1] * 20, [129, 127, 256, 1, 0, 2]]


@pytest.mark.parametrize("case", range(len(SIZES)))
def test_tile_table_covers_each_probed_pair_once(case):
    for seed in range(3):
        perm, off, probes = _table_case(seed, SIZES[case])
        slots, tiles = M.tile_table(probes, off)
        pairs = M.covered_pairs(slots, tiles, perm)
        want = [(q, int(r)) for q in range(probes.shape[0]) for r in M.union(probes[q], perm, off)]
        assert len(pairs) == len(set(pairs)) and sorted(pairs) == sorted(want)
        assert len(slots) % M.TILE == 0 and all(a % M.TILE == 0 for a, *_ in tiles)


def test_planted_bugs_are_caught():
    perm, off, probes = _table_case(0, SIZES[0])
    want = sorted((q, int(r)) for q in range(probes.shape[0]) for r in M.union(probes[q], perm, off))
    slots, tiles = M.tile_table(probes, off, bug="drop_last_tile")
    assert sorted(M.covered_pairs(slots, tiles, perm)) != want
    X, C, q, E, Ec, labels = _case(1)
    perm, off = M.build(labels, C.shape[0])
    probes = M.probe(Ec, 2)
    good = M.search(E, probes, perm, off, 300)
    bad_perm, bad_off = M.build(labels, C.shape[0], bug="cell_off_shift")
    assert not np.array_equal(M.search(E, probes, bad_perm, bad_off, 300)[1], good[1])
    # rows 0 and 1 tie; row 0 lies in the later list, so list positions order them the other way
    tp, to = M.build(np.array([1, 0, 1]), 2)
    tie = np.zeros((1, 3))
    both = np.array([[0, 1]])
    assert M.search(tie, both, tp, to, 3)[1].tolist() == [[0, 1, 2]]
    assert M.search(tie, both, tp, to, 3, bug="tie_by_position")[1].tolist() != [[0, 1, 2]]
    assert not np.array_equal(M.probe(Ec, 2, bug="probe_tie_larger"), probes)
    # the band: a query with a row exactly at the k-th group maximum's fp16 score minus 1.5 eps16 on the exact side
    F = np.zeros((1, 64), np.float32)
    F[0, :32] = 0.5
    F[0, 32] = np.float32(0.5 - 1.5 * BAND / 2)
    p1, o1 = np.arange(64), np.array([0, 64])
    assert 32 in M.candidates(F, np.zeros((1, 1), np.int64), p1, o1, 1, BAND)[0]
    assert 32 not in M.candidates(F, np.zeros((1, 1), np.int64), p1, o1, 1, BAND, bug="no_band")[0]
    r = np.random.RandomState(0)
    t_q = np.repeat(np.arange(q.shape[0]), 5)
    t_rows = r.randint(0, X.shape[0], t_q.shape[0])
    assert not np.array_equal(M.ranks(E, probes, perm, off, t_q, t_rows, bug="a_in_all_rows"),
                              M.ranks(E, probes, perm, off, t_q, t_rows))


def test_probe_range():
    Ec = np.zeros((2, 4))
    for bad in (0, 5):
        with pytest.raises(ValueError):
            M.probe(Ec, bad)


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "search.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+ivf_\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 8
    blocks += re.findall(r"Compiling entry function '(\w+conv_pers_kernelILi128ELi6ELi[67]E\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 10
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)


def test_ivf_argument_parsing():
    from dirb200.pipeline import ivf_params
    assert ivf_params([64, 8]) == dict(n_lists=64, nprobe=8, seed=0)
    assert ivf_params([5.0, 5.0]) == dict(n_lists=5, nprobe=5, seed=0)
    for bad in ([4], [4, 2, 1], [0, 1], [4, 0], [4.5, 2], [4, 5]):
        with pytest.raises(ValueError):
            ivf_params(bad)
    from dirtorch import test_dir
    for argv in (["--ivf", "4", "5"], ["--ivf", "4", "2", "--diffusion", "5", "3"], ["--ivf", "4"]):
        with pytest.raises(SystemExit):
            test_dir.test_dir_main(["--dataset", "Oxford5K", "--checkpoint", "none"] + argv)
