"""numpy model of the PCA statistics kernels (csrc/pca.cu) and the per-element bounds their results are held to.

gram_model follows the kernel's structure - 128 x 128 tiles on or above the diagonal, split-K over the rows with the
split rule of dirb200_gram_f64, 16-row K steps, partials added in split order and mirrored - so that the CPU suite can
show that the bound catches the mistakes such a kernel can make (tests/test_pca_host.py)."""
import numpy as np

U = 2.0 ** -53
GT, GK = 128, 32
GRAM_MAX_TILES, GRAM_SPLIT_ROWS = 2048, 1024        # pca.cu: 256 MiB of 128 x 128 fp64 partial tiles


def gamma(n):
    return n * U / (1 - n * U)


def gram_splits(n, d):
    """(splits, rows per split) of dirb200_gram_f64: a function of (N, D) only."""
    t = -(-d // GT)
    tiles = t * (t + 1) // 2
    s_want = min(GRAM_MAX_TILES // tiles, max(1, n // GRAM_SPLIT_ROWS))
    rows = -(-(-(-n // s_want)) // GK) * GK
    return -(-n // rows), rows


def centred(x, mean):
    return x.astype(np.float64) - np.asarray(mean, np.float64)


def gram_reference(x, mean, chunk=65536):
    """(G = a^T a, |a|^T |a|) in numpy fp64 with a = float64(x) - mean, accumulated over row chunks."""
    d = x.shape[1]
    g, ga = np.zeros((d, d)), np.zeros((d, d))
    for s in range(0, x.shape[0], chunk):
        a = centred(x[s:s + chunk], mean)
        g += a.T @ a
        aa = np.abs(a)
        ga += aa.T @ aa
    return g, ga


def gram_bound(n, ga):
    """|G_gpu - G_ref| <= 2 gamma(N + 4) sum_r |a_ri| |a_rj| (each of the two within gamma(N + 4) of the exact sum)."""
    return 2 * gamma(n + 4) * ga


def sums_bound(x):
    """|s_gpu - s_ref| <= 2 gamma(N) sum_r |x_rj| (both sums in fp64 in some order)."""
    return 2 * gamma(x.shape[0]) * np.abs(x.astype(np.float64)).sum(0)


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound (0 where both the difference and the bound are 0)."""
    diff = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(diff == 0, 0.0, diff / bound)
    return float(np.max(r)) if r.size else 0.0


def gram_model(x, mean, bug=None):
    """The kernel's Gram, in numpy.  bug: None, 'drop_kstep' (one 16-row K step of one tile skipped),
    'mirror_transposed' (an off-diagonal tile mirrored without transposing it), 'lose_last_split' (the last split's
    partials not added), 'mean_fp32' (the mean subtracted in fp32)."""
    n, d = x.shape
    t = -(-d // GT)
    s_cnt, rows = gram_splits(n, d)
    if bug == "mean_fp32":
        a = (x.astype(np.float32) - np.asarray(mean).astype(np.float32)).astype(np.float64)
    else:
        a = centred(x, mean)
    dp = t * GT
    a = np.pad(a, ((0, 0), (0, dp - d)))
    g = np.zeros((d, d))
    first = True
    for bi in range(t):
        for bj in range(bi, t):
            acc = np.zeros((GT, GT))
            for s in range(s_cnt):
                if bug == "lose_last_split" and s == s_cnt - 1:
                    continue
                part = np.zeros((GT, GT))
                for k0 in range(s * rows, min(n, (s + 1) * rows), 16):
                    if bug == "drop_kstep" and first and k0 == s * rows:
                        first = False
                        continue
                    blk = a[k0:min(n, k0 + 16)]
                    part += blk[:, bi * GT:(bi + 1) * GT].T @ blk[:, bj * GT:(bj + 1) * GT]
                acc += part
            i1, j1 = min(d, (bi + 1) * GT), min(d, (bj + 1) * GT)
            blk = acc[:i1 - bi * GT, :j1 - bj * GT]
            if bi == bj:
                up = np.triu(blk)
                g[bi * GT:i1, bj * GT:j1] = up + np.triu(up, 1).T
            else:
                g[bi * GT:i1, bj * GT:j1] = blk
                if bug == "mirror_transposed" and blk.shape[0] == blk.shape[1]:
                    g[bj * GT:j1, bi * GT:i1] = blk
                else:
                    g[bj * GT:j1, bi * GT:i1] = blk.T
    return g


def planted(n, d, lam, mean, seed=0, dtype=np.float32):
    """n x d rows whose centred fp64 covariance has (up to the rounding to dtype) exactly the eigenvalues lam (length
    min(n - 1, d), descending) on the random orthonormal basis q: x = mean + U diag(sqrt(lam (n - 1))) q^T with U
    orthonormal and orthogonal to the ones vector.  -> (x, q)."""
    r = np.random.RandomState(seed)
    k = len(lam)
    z = r.standard_normal((n, k))
    z -= z.mean(0)
    u, _ = np.linalg.qr(z)
    q, _ = np.linalg.qr(r.standard_normal((d, d)))
    x = np.asarray(mean, np.float64) + (u * np.sqrt(np.asarray(lam) * (n - 1))) @ q[:, :k].T
    return x.astype(dtype), q
