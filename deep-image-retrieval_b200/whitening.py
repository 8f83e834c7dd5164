"""Learn the PCA whitening that ``--whiten NAME`` applies (``checkpoint['pca'][NAME]``, a pickled sklearn PCA).

The reference only applies a whitening shipped with its checkpoints; fitting one means sklearn's ``PCA.fit`` on the
host.  Here the statistics come from the GPU in two passes over the rows (each streamed in chunks):

    1. column sums in fp64 (dirb200_col_sums_f64) -> mean = sums / N;
    2. the centred Gram G = (X - mean)^T (X - mean) on fp64 tensor cores (dirb200_gram_f64), C = G / (N - 1).

The eigendecomposition of C (D x D, independent of N) runs on the host in fp64 (numpy.linalg.eigh), and the
result is post-processed exactly as sklearn >= 1.5 does in ``_fit_full`` (``covariance_eigh`` branch): eigenvalues
descending and clipped at 0, ``svd_flip(u_based_decision=False)`` signs, variance ratios over all eigenvalues.  The
returned object is a real ``sklearn.decomposition.PCA`` so that the checkpoint stays loadable wherever sklearn is.
"""
from __future__ import annotations

import numpy as np
import torch

from . import inputs, ops


def _check_n_components(n_components, n, d):
    if n_components is None:
        return min(n, d)
    return inputs.check_int(n_components, "n_components", 1, min(n, d))


def pca_from_gram(n, sums, gram, n_components=None):
    """Host finalisation: (n rows, fp64 column sums (D,), centred fp64 Gram (D,D)) -> fitted sklearn PCA
    (whiten=True, svd_solver='covariance_eigh'), every attribute as sklearn's _fit_full computes it."""
    from sklearn.decomposition import PCA
    n = int(n)
    sums = np.asarray(sums, dtype=np.float64)
    gram = np.asarray(gram, dtype=np.float64)
    d = sums.shape[0]
    if n < 2:
        raise ValueError("a PCA fit needs at least 2 samples, got %d" % n)
    if gram.shape != (d, d):
        raise ValueError("Gram matrix of shape %s does not match %d features" % (gram.shape, d))
    k = _check_n_components(n_components, n, d)
    mean = sums / n
    if not (np.all(np.isfinite(mean)) and np.all(np.isfinite(gram))):
        raise ValueError("Input contains NaN or infinity.")
    cov = gram / (n - 1)
    lam, vec = np.linalg.eigh(cov)
    lam, vec = lam[::-1].copy(), vec[:, ::-1]
    lam[lam < 0.0] = 0.0
    comp = np.ascontiguousarray(vec.T)
    # svd_flip(u_based_decision=False): the largest |entry| of every component positive (first index on ties)
    signs = np.sign(comp[np.arange(d), np.argmax(np.abs(comp), axis=1)])
    comp *= signs[:, None]
    total = lam.sum()
    pca = PCA(n_components=n_components, whiten=True, svd_solver="covariance_eigh")
    pca.n_features_in_ = d
    pca.n_samples_ = n
    pca.n_components_ = k
    pca.mean_ = mean
    pca.components_ = comp[:k].copy()
    pca.explained_variance_ = lam[:k].copy()
    pca.explained_variance_ratio_ = lam[:k] / total
    pca.singular_values_ = np.sqrt(lam[:k] * (n - 1))
    pca.noise_variance_ = float(np.mean(lam[k:])) if k < min(n, d) else 0.0
    return pca


def fit_pca(X, n_components=None, chunk_rows=65536):
    """Fit PCA(n_components, whiten=True) on the GPU.  X: (N, D) CUDA tensor, CPU tensor, ndarray (a memmap works) or
    DescriptorStore; host rows are streamed chunk_rows at a time (read twice, once per pass) to the current CUDA
    device, a CUDA tensor is used on its own device.
    -> sklearn.decomposition.PCA equal to sklearn's own covariance_eigh fit of X in fp64 up to the rounding of the
    statistics (tests/test_gpu_pca.py states the bounds)."""
    src = inputs.Rows(X)
    n, d = src.n, src.d
    _check_n_components(n_components, max(n, 1), d)
    if n < 2:
        raise ValueError("a PCA fit needs at least 2 samples, got %d" % n)
    device = inputs.device(None, X)
    ops.require_gpu(device.index)
    if isinstance(X, torch.Tensor) and X.is_cuda:
        chunk_rows = n                                # a CUDA tensor as one view
    with torch.cuda.device(device):                   # the library launches on the current device's current stream
        sums = torch.zeros(d, dtype=torch.float64, device=device)
        for x in src.chunks(chunk_rows, device):
            ops.col_sums_f64(x, sums)
        sums_h = sums.cpu().numpy()
        if not np.all(np.isfinite(sums_h / n)):
            raise ValueError("Input contains NaN or infinity.")
        mean = sums / n
        gram = torch.zeros((d, d), dtype=torch.float64, device=device)
        for x in src.chunks(chunk_rows, device):
            ops.gram_f64(x, mean, gram)
        gram_h = gram.cpu().numpy()
    return pca_from_gram(n, sums_h, gram_h, n_components)
