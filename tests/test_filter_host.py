"""Filtered exact search on the CPU (DESIGN.md section 4.13): allow_rows against numpy.packbits, the model's seed rule
(F2) and shard windows (F6) against plain loops, the model against the exact filtered top-k (F5) including the shard
protocols, four planted bugs it must catch, argument validation, and the new kernels' compiler statistics."""
import os
import re

import numpy as np
import pytest
import torch

import filter_model as FM
import search_model as SM
from conftest import REPO


def _bit(words_row, b):
    return (int(words_row[b >> 5]) >> (b & 31)) & 1


def _data(n, nq, d=32, seed=0):
    r = np.random.RandomState(seed)
    db = r.standard_normal((n, d)).astype(np.float32)
    db /= np.linalg.norm(db, axis=1, keepdims=True)
    q = r.standard_normal((nq, d)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return db, q


@pytest.mark.parametrize("shape", [(1,), (31,), (32,), (33,), (3, 100), (2, 5, 64)])
def test_allow_rows_matches_packbits(shape):
    from dirb200 import ops
    mask = np.random.RandomState(len(shape)).rand(*shape) < 0.5
    words = ops.allow_rows(torch.from_numpy(mask)).numpy()
    assert words.dtype == np.int32 and words.shape == shape[:-1] + ((shape[-1] + 31) // 32,)
    assert np.array_equal(words.view(np.uint32), FM.pack(mask))
    n = shape[-1]
    pad = np.zeros(shape[:-1] + (32 * ((n + 31) // 32),), bool)
    pad[..., :n] = mask
    ref = np.packbits(pad, axis=-1, bitorder="little").view("<u4")
    assert np.array_equal(words.view(np.uint32), ref)


def test_allow_rows_rejects_non_bool():
    from dirb200 import ops
    with pytest.raises(ValueError):
        ops.allow_rows(torch.zeros(10, dtype=torch.int32))


@pytest.mark.parametrize("seed", range(6))
def test_seed_rule_and_windows_equal_loops(seed):
    r = np.random.RandomState(seed)
    n_global = int(r.randint(1, 300))
    bit0 = int(r.randint(0, n_global))
    n = int(r.randint(0, n_global - bit0 + 1))
    nq = int(r.randint(1, 5))
    mask = r.rand(nq, n_global) < [0.97, 0.5, 0.1][seed % 3]
    words = FM.pack(mask)
    A = FM.window(words, bit0, n)
    for qi in range(nq):
        assert [bool(_bit(words[qi], bit0 + i)) for i in range(n)] == list(A[qi])
    S = int(r.randint(1, 80))
    rows = []
    for i in range(n):
        if all(_bit(words[qi], bit0 + i) for qi in range(nq)) and len(rows) < S:
            rows.append(i)
    assert list(FM.seed_rows(A, S)) == rows
    shared = FM.window(words[0], bit0, n)                 # a (W,) set is one row shared by every query
    assert np.array_equal(shared[0], A[0])


def _allow_cases(n, nq, r):
    yield "all", np.ones((n,), bool)
    for frac in (0.5, 0.1, 0.01):
        yield "rand%g" % frac, r.rand(n) < frac
    blk = np.zeros(n, bool)
    blk[-n // 10:] = True
    yield "block_end", blk
    one = np.zeros(n, bool)
    one[n // 3] = True
    yield "one_row", one
    yield "empty", np.zeros(n, bool)
    few = np.zeros(n, bool)
    few[r.choice(n, 7, replace=False)] = True
    yield "fewer_than_k", few
    yield "per_query", r.rand(nq, n) < 0.3
    disj = np.zeros((nq, n), bool)
    for i in range(nq):
        disj[i, i::nq] = True
    yield "disjoint", disj
    loo = np.ones((nq, n), bool)
    loo[np.arange(nq), np.arange(nq)] = False
    yield "self_exclusion", loo


@pytest.mark.parametrize("bounds", [None, [(0, 700), (700, 701), (701, 701), (701, 2000)],
                                    [(0, 333), (333, 1000), (1000, 1777), (1777, 2000)]])
@pytest.mark.parametrize("peer", [False, True])
def test_model_equals_exact_filtered_topk(bounds, peer):
    db, q = _data(2000, 6, seed=1)
    r = np.random.RandomState(2)
    for k in (1, 10, 40):
        for name, mask in _allow_cases(2000, 6, r):
            words = FM.pack(mask)
            es, ei = FM.exact_filtered_topk(q, db, k, words)
            ms, mi = FM.filtered_search(q, db, k, words, sample_rows=256, bounds=bounds, peer=peer, cand_cap=300)
            assert np.array_equal(mi, ei), (name, k)
            assert np.array_equal(ms, es), (name, k)


def test_all_bits_equal_unfiltered_model():
    db, q = _data(3000, 5, seed=3)
    words = FM.pack(np.ones(3000, bool))
    for k in (1, 50, 100):
        fs, fi = FM.filtered_search(q, db, k, words, sample_rows=512)
        us, ui = SM.exact_topk(q, db, k)
        assert np.array_equal(fi, ui) and np.array_equal(fs, us)


def _trap():
    """Allowed rows far from the queries, disallowed rows (every row of word 0, the queries' own rows) close to them."""
    db, q = _data(1500, 4, seed=4)
    near = q[:, None, :] + 0.05 * np.random.RandomState(5).standard_normal((4, 40, q.shape[1])).astype(np.float32)
    near = (near / np.linalg.norm(near, axis=-1, keepdims=True)).reshape(-1, q.shape[1])
    db = np.concatenate([near, db]).astype(np.float32)        # rows 0..159 close to the queries
    mask = np.ones((4, db.shape[0]), bool)
    for i in range(4):
        mask[i, 40 * i:40 * i + 40] = False                    # query i excludes its own near rows
    mask[:, 63] = False                                        # a word-edge bit
    mask[:, 200:232] = False
    mask[1:, 31] = False                                       # row 31 excluded for all but query 0
    return q, db, mask


@pytest.mark.parametrize("bug", ["seed_outside", "no_bit", "bit0", "word_edge"])
def test_planted_bugs_are_caught(bug):
    q, db, mask = _trap()
    words = FM.pack(mask)
    es, ei = FM.exact_filtered_topk(q, db, 30, words)
    caught = False
    for bounds in (None, [(0, 100), (100, 777), (777, db.shape[0])]):
        ms, mi = FM.filtered_search(q, db, 30, words, sample_rows=256, bounds=bounds)
        assert np.array_equal(mi, ei)                           # the correct model passes
        bs, bi = FM.filtered_search(q, db, 30, words, sample_rows=256, bounds=bounds, bug=bug)
        caught |= not np.array_equal(bi, ei)
    assert caught, bug


def test_argument_validation():
    from dirb200 import ops
    with pytest.raises(ValueError):
        ops.allow_rows(np.ones(4, bool))
    with pytest.raises(TypeError):
        ops.allow_exclude(torch.zeros(4, dtype=torch.int32), 2, [[1], [2]])     # not a CUDA tensor


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "search.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    pat = r"Compiling entry function '(\w+(?:allow_\w+_kernel\w*|conv_pers_kernelILi128ELi6ELi8E\w*))'.*?\n.*?\n(.*?)\n"
    blocks = re.findall(pat, text)
    names = sorted(set(re.sub(r".*?(allow_\w+_kernel|conv_pers_kernel).*", r"\1", n) for n, _ in blocks))
    assert names == ["allow_and_kernel", "allow_exclude_kernel", "allow_gather_kernel", "allow_kth_kernel",
                     "allow_seed_rows_kernel", "conv_pers_kernel"], names
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)
