"""numpy model of csrc/aploss.cu and the seeded score / label generators the AP-loss tests share.

The model takes every decision the kernels take, on the same fp32 values: v = fl32(fmaf(w, x, b)) (emulated exactly:
an fp64 product is exact, and the fp64 sum is rounded to odd before the fp32 rounding, so nothing rounds twice), the
candidate bins around rint(v_1), q rounded to nearest in units of 2^-32, int64 sums, and the fp64 finalisation in bin
order.  Keyword switches plant the bugs the tests must catch.  The fp64 restatement of the reference the model is
checked against lives apart from it, in tests/aploss_oracle.py."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import synthdata as synth  # noqa: E402

U64 = 2.0 ** -53
FIX = 2.0 ** 32


def gamma(k):
    return k * U64 / (1 - k * U64)


def table(nq, lo, hi):
    """The reference's quantiser (loss.py:29-41) as 2nq fp32 weights and 2nq fp32 biases."""
    a = (nq - 1) / (hi - lo)
    w = np.empty(2 * nq, np.float32)
    w[:nq] = -a
    w[nq:] = a
    b = np.concatenate([a * lo + np.arange(nq, 0, -1), np.arange(2 - nq, 2, 1) - a * lo]).astype(np.float32)
    w[0] = w[-1] = 0
    b[0] = b[-1] = 1
    return w, b


def fmaf(w, x, b):
    """fl32(w * x + b) with a single rounding, elementwise (fp32 inputs)."""
    p = np.asarray(w, np.float64) * np.asarray(x, np.float64)   # exact: 24 x 24 bits
    b = np.asarray(b, np.float64)
    s = p + b
    bv = s - p
    e = (p - (s - bv)) + (b - bv)                           # TwoSum: s + e == p + b exactly
    even = (s.view(np.int64) & 1) == 0
    odd = np.where((e != 0) & even, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return odd.astype(np.float32)


def candidates(x, w, b, nq):
    """k (rint of v_1, clipped to [-1, nq]) and, for the bins k-1, k, k+1: the bin index, whether it exists, the
    pre-clamp value min(v_j, v_{j+nq}) and the branch the min takes (-1 low line, +1 high line, 0 tie)."""
    x = np.asarray(x, np.float32)
    p = fmaf(w[1], x, b[1])
    k = np.rint(np.clip(p, -1, nq)).astype(np.int64)
    out = []
    for s in range(3):
        j = k - 1 + s
        ok = (j >= 0) & (j < nq)
        jj = np.clip(j, 0, nq - 1)
        vlo = fmaf(w[jj], x, b[jj])
        vhi = fmaf(w[jj + nq], x, b[jj + nq])
        out.append((jj, ok, np.minimum(vlo, vhi), np.sign(vhi.astype(np.float64) - vlo)))
    return k, out


def histogram(x, label, w, b, nq, round_fix=True):
    """int64 [N][2nq+1]: c, cp and the positive count, in units of 2^-32 (round_fix=False truncates instead)."""
    N, M = x.shape
    h = np.zeros((N, 2 * nq + 1), np.int64)
    lab = np.asarray(label) != 0
    rows = np.repeat(np.arange(N), M).reshape(N, M)
    _, cands = candidates(x, w, b, nq)
    for jj, ok, m, _ in cands:
        q = np.maximum(m, np.float32(0)).astype(np.float64) * FIX
        f = np.where(ok, np.rint(q) if round_fix else np.floor(q), 0).astype(np.int64)
        np.add.at(h, (rows, jj), f)
        np.add.at(h, (rows, nq + jj), np.where(lab, f, 0))
    h[:, 2 * nq] = lab.sum(1).astype(np.int64) << 32
    return h


def finalize(h, nq, mode, eps=None, rev_shift=0):
    """fp64 AP (N,), G (N,2nq) and the magnitudes that bound their rounding errors, in the kernel's order.
    mode 'ap' / 'tap' / 'taps'.  rev_shift=1 plants an off-by-one in the reverse cumulative sums."""
    h = np.asarray(h, np.int64)
    c = h[:, :nq].astype(np.float64) / FIX
    cp = h[:, nq:2 * nq].astype(np.float64) / FIX
    Np = h[:, 2 * nq].astype(np.float64) / FIX
    N = h.shape[0]
    C = np.cumsum(c, 1)
    P = np.cumsum(cp, 1)
    C1 = np.concatenate([np.zeros((N, 1)), C[:, :-1]], 1)
    P1 = np.concatenate([np.zeros((N, 1)), P[:, :-1]], 1)
    G = np.zeros((N, 2 * nq))
    Gm = np.zeros((N, 2 * nq))

    def rsum(v, inclusive=True):   # sum_{j >= k} (inclusive) or sum_{j > k}, k along axis 1
        r = np.cumsum(v[:, ::-1], 1)[:, ::-1]
        r = r if inclusive else np.concatenate([r[:, 1:], np.zeros((N, 1))], 1)
        if rev_shift:
            r = np.concatenate([r[:, rev_shift:], np.zeros((N, rev_shift))], 1)
        return r

    with np.errstate(divide="ignore", invalid="ignore"):
        if mode == "ap":
            e = 1e-16 if eps is None else eps
            S = P[:, -1:]
            d = e + C
            A = P / d
            u = cp / S
            ap = (A * u).sum(1)
            G[:, :nq] = -rsum(u * A / d)
            G[:, nq:] = A / S + rsum(u / d) - ap[:, None] / S
            mag_ap = np.abs(A * u).sum(1)
            Gm[:, :nq] = rsum(np.abs(u * A / d))
            Gm[:, nq:] = np.abs(A / S) + rsum(np.abs(u / d)) + np.abs(ap[:, None] / S)
        elif mode == "taps":
            D = C1 + C + 1
            Nu = P1 + P + 1
            apj = cp * Nu / D / Np[:, None]
            ap = apj.sum(1)
            G[:, :nq] = -apj / D - 2 * rsum(apj / D, False)
            G[:, nq:] = (Nu + cp) / (D * Np[:, None]) + 2 * rsum(cp / (D * Np[:, None]), False)
            mag_ap = np.abs(apj).sum(1)
            Gm[:, :nq] = np.abs(apj / D) + 2 * rsum(np.abs(apj / D), False)
            Gm[:, nq:] = np.abs((Nu + cp) / (D * Np[:, None])) + 2 * rsum(np.abs(cp / (D * Np[:, None])), False)
        else:
            e = 1e-8 if eps is None else eps
            hc, hp = c - 1, cp - 1
            den = np.maximum(hc, 0) + e
            r = np.maximum(hp, 0) / den
            L = np.log((C + 1) / (C1 + 1))
            B = P1 + 1 - r * (C1 + 1)
            T = c * r + B * L
            E = cp / (c + e) / Np[:, None]
            apj = cp * T / (c + e) / Np[:, None]
            ap = apj.sum(1)
            alpha = E * B / (C + 1)
            beta = E * (-r * L - B / (C1 + 1))
            rho = E * (c - (C1 + 1) * L)
            drc = np.where(hc >= 0, -r / den, 0.0)
            drp = np.where(hp >= 0, 1 / den, 0.0)
            G[:, :nq] = -apj / (c + e) + E * r + rho * drc + rsum(alpha) + rsum(beta, False)
            G[:, nq:] = T / ((c + e) * Np[:, None]) + rho * drp + rsum(E * L, False)
            # magnitudes: every subtraction taken as a sum of absolute values, |L| widened by 1 (log's own rounding
            # and that of its argument are absolute errors of about one ulp of 1)
            La = np.abs(L) + 1
            Ba = P1 + 1 + r * (C1 + 1)
            Ta = c * r + Ba * La
            Ea = np.abs(E)
            mag_ap = np.abs(cp * Ta / (c + e) / Np[:, None]).sum(1)
            rhoa = Ea * (c + (C1 + 1) * La)
            Gm[:, :nq] = (Ea * Ta / (c + e) + Ea * r + rhoa * np.abs(drc) + rsum(Ea * Ba / (C + 1))
                          + rsum(Ea * (r * La + Ba / (C1 + 1)), False))
            Gm[:, nq:] = Ta / ((c + e) * np.abs(Np[:, None])) + rhoa * np.abs(drp) + rsum(Ea * La, False)
    return ap, G, mag_ap, Gm


def bounds(nq, mag_ap, Gm):
    """Kernel vs model, both fp64 from the same histogram: at most ~4nq + 16 roundings along any path (the cumulative
    sums, the reverse sums, a handful per term), each relative to the magnitude of what it rounds; 2 gamma covers
    both sides.  The fp32 AP adds one rounding."""
    k = 4 * nq + 16
    return 2 * gamma(k) * mag_ap, 2 * gamma(k) * Gm


def backward(x, label, w, b, nq, G, grad_ap, clamp_ge=True, tie_split=True):
    """dx (fp32) from the coefficients G, and a bound-magnitude: |sum of terms| * |grad_ap|."""
    x = np.asarray(x, np.float32)
    lab = np.asarray(label) != 0
    N = x.shape[0]
    rows = np.arange(N)[:, None]
    _, cands = candidates(x, w, b, nq)
    s = np.zeros(x.shape)
    mag = np.zeros(x.shape)
    for jj, ok, m, br in cands:
        wlo = w[jj].astype(np.float64)
        whi = w[jj + nq].astype(np.float64)
        if tie_split:
            slope = np.where(br > 0, wlo, np.where(br < 0, whi, 0.5 * (wlo + whi)))
        else:
            slope = np.where(br >= 0, wlo, whi)
        act = ok & ((m >= 0) if clamp_ge else (m > 0))
        gc = G[rows, jj]
        gp = G[rows, nq + jj]
        t = np.where(act, np.where(lab, gc + gp, gc) * slope, 0.0)
        s += t
        mag += np.abs(t)
    g = np.asarray(grad_ap, np.float64)[:, None]
    with np.errstate(invalid="ignore"):
        dx = (g * s).astype(np.float32)
    return dx, np.abs(g) * mag


# ---- seeded inputs ----

def make_scores(seed, N, M, nq, lo, hi, kind):
    """x (N,M) fp32 and labels (N,M) uint8 (about 10 % positives, row 0 guaranteed one).  kind: 'uniform' in
    [lo, hi]; 'outside' with 20 % beyond it; 'concentrated' with 99 % inside one bin; 'kinks' on bin centres and
    edges (every bin's peak and the midpoints between peaks)."""
    r = synth._rs(seed, "aploss.%s.%d.%d.%d" % (kind, N, M, nq))
    gap = hi - lo
    if kind == "uniform":
        x = r.uniform(lo, hi, (N, M))
    elif kind == "outside":
        x = r.uniform(lo, hi, (N, M))
        o = r.uniform(0, 1, (N, M)) < 0.2
        x[o] = np.where(r.uniform(0, 1, o.sum()) < 0.5, lo - r.uniform(0, gap, o.sum()), hi + r.uniform(0, gap, o.sum()))
    elif kind == "concentrated":
        centre = hi - gap * (nq // 3 + 0.3) / (nq - 1)
        x = centre + r.uniform(-0.1, 0.1, (N, M)) * gap / (nq - 1)
        o = r.uniform(0, 1, (N, M)) < 0.01
        x[o] = r.uniform(lo, hi, o.sum())
    elif kind == "kinks":
        pts = lo + gap * np.arange(0, 2 * (nq - 1) + 1) / (2 * (nq - 1))
        x = pts[r.randint(0, len(pts), (N, M))]
    else:
        raise ValueError(kind)
    lab = (r.uniform(0, 1, (N, M)) < 0.1).astype(np.uint8)
    lab[:, 0] = 1
    return x.astype(np.float32), lab


def fixed_point_case(M=4096):
    """Scores whose bin values are exact and have a fractional part of 3/4 in units of 2^-32, with their exact bin sums
    (in units of 2^-32).  nq = 17 on [0, 1]: a = 16, every table value is exact, and x = 3 * 2^-38 gives bin 15
    exactly 16 x = 0.75 * 2^-32 and bin 16 1 - 16 x, which rounds to 1 in fp32."""
    x = np.full((1, M), 3 * 2.0 ** -38, np.float32)
    lab = np.zeros((1, M), np.uint8)
    lab[0, ::2] = 1
    exact = np.zeros(2 * 17 + 1)
    exact[15] = 0.75 * M
    exact[16] = FIX * M
    exact[17 + 15] = 0.75 * (M // 2)
    exact[17 + 16] = FIX * (M // 2)
    exact[34] = FIX * (M // 2)
    return x, lab, exact


def fixed_point_error(h, exact, M):
    """max over bins of |hist - exact sum| in units of the rounding bound M / 2 (half a unit per element)."""
    return float(np.max(np.abs(h[0].astype(np.float64) - exact)) / (M / 2))
