"""Reference restatements for the label-count tests: threshold counts from the dense exact scores, and the epilogue's
rounding-boundary rule of dirb200_index_count_ge."""
import numpy as np

from oracle import dir_oracle as O


def ge_counts(Q, DB, t_off, thr, skip=None):
    """count[t] = number of database rows r != skip[q] with fl32(exact score <Q[q], DB[r]>) >= thr[t]."""
    Q, DB = np.asarray(Q), np.asarray(DB)
    out = np.zeros(len(thr), dtype=np.int64)
    for q in range(len(t_off) - 1):
        if t_off[q] == t_off[q + 1]:
            continue
        row = O.scores_exact(Q[q:q + 1], DB)[0].astype(np.float32)
        if skip is not None and skip[q] >= 0:
            row = np.delete(row, int(skip[q]))
        srt = np.sort(row)
        seg = np.asarray(thr[t_off[q]:t_off[q + 1]], dtype=np.float32)
        out[t_off[q]:t_off[q + 1]] = len(srt) - np.searchsorted(srt, seg, side="left")
    return out


def boundary(s):
    """m = (pred32(s) + s) / 2 in fp64 (exact): fl32(e) >= s  <=>  e > m, or e == m and s has an even significand."""
    s = np.float32(s)
    return (float(np.nextafter(s, np.float32(-np.inf))) + float(s)) / 2.0


def even_significand(s):
    return (int(np.asarray(s, dtype=np.float32).view(np.uint32)) & 1) == 0


def decide(x, eps, s):
    """The epilogue's decision for a tensor-core score x known to lie within eps of the exact score:
    True = reaches s for certain, False = does not, None = band (re-scored exactly)."""
    m = boundary(s)
    if x - eps > m:
        return True
    if x + eps < m:
        return False
    return None
