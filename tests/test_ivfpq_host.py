"""IVF-PQ on the CPU (DESIGN.md section 4.11): the model of tests/ivfpq_model.py against dense restatements of rules
P3-P8, rule P7's identities, six planted bugs, the --pq / --refine parsing, the chunked build's bookkeeping, the
workspace sizes and spills of the new kernels."""
import os
import re

import numpy as np
import pytest

import ivf_model as IM
import ivfpq_model as P
import kmeans_model as KM
from conftest import REPO


def _unit(x):
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _case(seed, n=600, d=64, K=6, nq=5, M=8, it=2):
    r = np.random.RandomState(seed)
    C = _unit(r.standard_normal((K, d)))
    X = _unit(C[r.randint(0, K, n)] + 0.4 * r.standard_normal((n, d)) / 8)
    X[7] = X[3]                                   # equal codes and equal scores: ties go to the smaller row
    q = _unit(C[r.randint(0, K, nq)] + 0.4 * r.standard_normal((nq, d)) / 8)
    Ex, Ec = KM.exact_scores(X, C), KM.exact_scores(q, C)
    labels = KM.assign(Ex)[0]
    perm, off = IM.build(labels, K)
    CBs, _ = P.train(X, C, labels, M, 300, it, seed)
    codes = P.encode(P.residuals(X, C, labels), CBs)[perm]
    T = P.tables(q, CBs)
    return dict(X=X, C=C, q=q, E=KM.exact_scores(q, X), Ec=Ec, labels=labels, perm=perm, off=off, CBs=CBs, codes=codes,
                T=T, K=K)


@pytest.fixture(scope="module")
def case():
    return _case(0)


def test_codes_equal_brute_force_argmin(case):
    S = P.residuals(case["X"], case["C"], case["labels"])[:40, :8]
    CB = case["CBs"][0]
    want = []
    for s in S:
        dist = [sum((float(np.float64(s[t]) - np.float64(c[t]))) ** 2 for t in range(8)) for c in CB]
        want.append(min(range(256), key=lambda j: (dist[j], j)))
    assert P.nearest(S, CB).tolist() == want


def test_codeword_ties_go_to_the_smaller_index():
    CB = np.zeros((256, 4), np.float32)
    CB[:, 0] = np.arange(256)
    CB[9] = CB[3]
    S = CB[[3, 9, 200]]
    assert P.nearest(S, CB).tolist() == [3, 3, 200]
    assert P.nearest(S, CB, "tie_larger").tolist() == [9, 9, 200]


def test_update_keeps_empty_codewords():
    r = np.random.RandomState(1)
    Rs = r.standard_normal((300, 8)).astype(np.float32)
    CBs = r.standard_normal((1, 256, 8)).astype(np.float32)
    codes = np.zeros((300, 1), np.uint8)
    codes[::2, 0] = 5
    out, empty = P.update(Rs, codes, CBs)
    assert empty == 254
    assert np.array_equal(out[0, 1:5], CBs[0, 1:5])
    assert np.array_equal(out[0, 5], (Rs[::2].astype(np.float64).sum(0) / 150).astype(np.float32)) or \
        np.abs(out[0, 5] - Rs[::2].mean(0)).max() < 1e-6


def test_adc_equals_float32_loop(case):
    c = 2
    seg = slice(case["off"][c], case["off"][c + 1])
    codes = case["codes"][seg]
    T = case["T"][0]
    got = P.adc(T, np.float32(case["Ec"][0, c]), codes)
    for i in range(codes.shape[0]):
        s = np.float32(case["Ec"][0, c])
        for m in range(codes.shape[1]):
            s = np.float32(s + T[m, codes[i, m]])
        assert got[i] == s


def test_tables_equal_per_entry_sums(case):
    q, CBs, T = case["q"], case["CBs"], case["T"]
    for m, j in ((0, 0), (3, 17), (7, 255)):
        acc = 0.0
        for t in range(8):
            acc += float(q[1, m * 8 + t]) * float(CBs[m, j, t])
        assert T[1, m, j] == np.float32(acc)


@pytest.mark.parametrize("R", [1, 7, 40, 10000])
def test_search_equals_full_sort(case, R):
    probes = IM.probe(case["Ec"], 3)
    k = min(R, 5)
    sc, ix, cands = P.search(case["E"], case["T"], case["Ec"], probes, case["codes"], case["perm"], case["off"], k, R)
    for q in range(probes.shape[0]):
        rows, a, _ = P.union_adc(case["T"][q], probes[q], case["Ec"][q], case["codes"], case["perm"], case["off"])
        full = sorted(zip(rows.tolist(), a.tolist()), key=lambda p: (-p[1], p[0]))[:R]
        cq = [r for r, _ in full]
        assert sorted(cands[q].tolist()) == sorted(cq)
        best = sorted(cq, key=lambda r: (-case["E"][q, r], r))[:k]
        assert ix[q, :len(best)].tolist() == best
        assert (ix[q, len(best):] == -1).all()


def test_identities_of_p7(case):
    E, K = case["E"], case["K"]
    for nprobe in (1, 3):
        probes = IM.probe(case["Ec"], nprobe)
        want = IM.search(E, probes, case["perm"], case["off"], 9)
        got = P.search(E, case["T"], case["Ec"], probes, case["codes"], case["perm"], case["off"], 9, E.shape[1])
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    probes = IM.probe(case["Ec"], K)
    got = P.search(E, case["T"], case["Ec"], probes, case["codes"], case["perm"], case["off"], 9, E.shape[1])
    order = np.lexsort((np.broadcast_to(np.arange(E.shape[1]), E.shape), -E), axis=1)[:, :9]
    assert np.array_equal(got[1], order)


def test_rank_model_equals_dense_restatement(case):
    probes = IM.probe(case["Ec"], 2)
    _, _, cands = P.search(case["E"], case["T"], case["Ec"], probes, case["codes"], case["perm"], case["off"], 5, 20)
    t_q = np.repeat(np.arange(5), 6)
    t_rows = np.random.RandomState(3).randint(0, case["E"].shape[1], 30)
    got = P.ranks(case["E"], cands, t_q, t_rows)
    for i, (q, t) in enumerate(zip(t_q, t_rows)):
        cq = sorted(cands[q].tolist(), key=lambda r: (-case["E"][q, r], r))
        rest = sorted(set(range(case["E"].shape[1])) - set(cq), key=lambda r: (-case["E"][q, r], r))
        assert got[i] == (cq + rest).index(t)
    # with C_q = R(q) the ranks are rule I7's
    allc = [IM.union(p, case["perm"], case["off"]) for p in probes]
    assert np.array_equal(P.ranks(case["E"], allc, t_q, t_rows),
                          IM.ranks(case["E"], probes, case["perm"], case["off"], t_q, t_rows))


def test_planted_bugs_are_caught():
    c = _case(4, it=1)
    X, C, labels = c["X"], c["C"], c["labels"]
    Rs = P.residuals(X, C, labels)
    caught = set()
    # distances: FMA and the tie rule move codes
    for bug in ("fma", "tie_larger"):
        CB = c["CBs"][0].copy()
        CB[11] = CB[10]                         # a planted tie
        S = np.concatenate([Rs[:, :8], CB[10:11]])
        if not np.array_equal(P.nearest(S, CB, bug), P.nearest(S, CB)) or \
                not np.array_equal(P.distances(S, CB, bug), P.distances(S, CB)):
            caught.add(bug)
    qq, cbs = np.zeros((1, 512), np.float32), np.ones((8, 256, 64), np.float32)
    qq[0, :3], cbs[0, 0, :3] = (1, 2 ** 30, 2 ** 30), (1, 2 ** 30, -2 ** 30)   # 1 + 2^60 - 2^60: 0 forward, 1 backward
    if not np.array_equal(P.tables(qq, cbs, "table_order"), P.tables(qq, cbs)):
        caught.add("table_order")
    probes = IM.probe(c["Ec"], 2)
    ref = P.search(c["E"], c["T"], c["Ec"], probes, c["codes"], c["perm"], c["off"], 5, 12)
    for bug in ("no_list_term", "cand_tie_position", "refine_adc"):
        codes = c["codes"]
        if bug == "cand_tie_position":          # rows whose ADC scores tie, listed against row order
            codes = codes.copy()
            codes[:] = codes[0]
        base = P.search(c["E"], c["T"], c["Ec"], probes, codes, c["perm"][::-1].copy() if bug == "cand_tie_position"
                        else c["perm"], c["off"], 5, 12)
        got = P.search(c["E"], c["T"], c["Ec"], probes, codes, c["perm"][::-1].copy() if bug == "cand_tie_position"
                       else c["perm"], c["off"], 5, 12, bug)
        if not (np.array_equal(got[1], base[1]) and all(np.array_equal(a, b) for a, b in zip(got[2], base[2]))):
            caught.add(bug)
    assert ref is not None
    assert caught == {"fma", "tie_larger", "table_order", "no_list_term", "cand_tie_position", "refine_adc"}


def test_chunk_plan_covers_every_row_once():
    from dirb200.ivfpq import _plan
    train = np.sort(np.random.RandomState(0).choice(1000, 300, replace=False))
    for cr in (1, 7, 333, 1000, 5000):
        plan = _plan(1000, cr, train)
        assert plan[0][0] == 0 and plan[-1][1] == 1000 and len(plan) == -(-1000 // cr)
        assert all(p[1] == nxt[0] and p[3] == nxt[2] for p, nxt in zip(plan, plan[1:]))
        assert plan[0][2] == 0 and plan[-1][3] == 300
        for a, b, lo, hi in plan:
            assert ((train[lo:hi] >= a) & (train[lo:hi] < b)).all()


def test_pq_argument_parsing():
    from dirb200.pipeline import ivf_params, pq_params
    ivf = ivf_params([64, 8])
    assert pq_params(ivf, None, None) == ivf
    assert pq_params(ivf, 32, None) == dict(ivf, pq=32, refine=400)
    assert pq_params(ivf, 8, 50) == dict(ivf, pq=8, refine=50)
    for bad in ((None, 8, None), (ivf, None, 40), (ivf, 12, None), (ivf, 8, 0)):
        with pytest.raises(ValueError):
            pq_params(*bad)
    from dirtorch import test_dir
    for argv in (["--pq", "8"], ["--ivf", "4", "2", "--refine", "9"], ["--ivf", "4", "2", "--pq", "7"]):
        with pytest.raises(SystemExit):
            test_dir.test_dir_main(["--dataset", "Oxford5K", "--checkpoint", "none"] + argv)


def test_search_workspace_sizes_are_pinned():
    from dirb200 import lib
    f = lib.raw("dirb200_pq_search_ws_bytes")
    table = [(1, 0, 1, 41984), (1, 1, 1, 41984), (1, 1000, 100, 49664), (1, 1000, 2048, 49664),
             (1, 1000, 2049, 90624), (70, 131072, 400, 3916544), (1000, 1048576, 400, 49352960), (0, 5, 5, 0)]
    assert [(*row[:3], f(*row[:3])) for row in table] == table


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "pq.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+pq_\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 6
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
