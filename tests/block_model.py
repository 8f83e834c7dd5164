"""numpy model of the block primitives in deep-image-retrieval_b200/csrc/block.cuh, written from what the header promises
rather than from how it computes it: the result order, the k-th largest key, inclusive sums, the rank of an entry in a
sorted run, and the merge of two runs."""
import numpy as np


def ranks_before(sa, ia, sb, ib):
    """(sa, ia) comes first in the result order: score descending, ties to the lower index, -0 == +0."""
    sa, sb = np.asarray(sa, np.float64), np.asarray(sb, np.float64)
    ia, ib = np.asarray(ia, np.int64), np.asarray(ib, np.int64)
    return (sa > sb) | ((sa == sb) & (ia < ib))


def result_order(scores, idx):
    """The permutation that puts (scores, idx) in the result order (numpy compares -0 and +0 as equal)."""
    return np.lexsort((np.asarray(idx, np.int64), -np.asarray(scores, np.float64)))


def float_total_order(x):
    """The permutation sorting fp32 values ascending with -0 just below +0 (no NaNs)."""
    x = np.asarray(x, np.float32)
    return np.lexsort((~np.signbit(x), x))


def kth_largest(keys, k):
    """The k-th largest of n unsigned keys, 1 <= k <= n, duplicates counted."""
    assert 1 <= k <= len(keys)
    return np.sort(keys)[-k]


def kth_largest_float(x, k):
    """The k-th largest fp32 value in the order of float_total_order."""
    x = np.asarray(x, np.float32)
    return x[float_total_order(x)[-k]]


def inclusive_sum(v, axis=-1):
    """Inclusive sums along axis in int64 / uint64 (uint64 wraps modulo 2^64), and the totals."""
    v = np.asarray(v)
    wide = v.astype(np.uint64 if v.dtype.kind == "u" else np.int64)
    incl = np.cumsum(wide, axis=axis, dtype=wide.dtype)
    return incl, np.take(incl, [-1], axis=axis)


def rank_in_run(sc, ix, s, i):
    """The number of valid entries (index >= 0) of the run (sc, ix) that rank before (s, i)."""
    sc, ix = np.asarray(sc, np.float64), np.asarray(ix, np.int64)
    return int(np.count_nonzero((ix >= 0) & ranks_before(sc, ix, s, i)))


def merge(a_sc, a_ix, b_sc, b_ix):
    """Two runs merged: their concatenation in the result order."""
    sc, ix = np.concatenate([a_sc, b_sc]), np.concatenate([a_ix, b_ix])
    p = result_order(sc, ix)
    return sc[p], ix[p]
