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

from . import ops
from .store import DescriptorStore


def _n_rows_dim(X):
    if isinstance(X, DescriptorStore):
        return X.n_rows, X.dim
    shape = tuple(X.shape)
    if len(shape) != 2:
        raise ValueError("expected a 2-D (n_samples, n_features) array, got shape %s" % (shape,))
    return shape


def _chunks(X, chunk_rows, device):
    """(N, D) rows of X as contiguous fp32 tensors on `device`, chunk_rows at a time (a CUDA tensor as one view)."""
    if isinstance(X, torch.Tensor) and X.is_cuda:
        x = X.to(device, torch.float32).contiguous()
        yield x
        return
    n = _n_rows_dim(X)[0]
    for s in range(0, n, chunk_rows):
        e = min(n, s + chunk_rows)
        if isinstance(X, DescriptorStore):
            block = torch.from_numpy(X.read_rows(s, e))
        elif isinstance(X, torch.Tensor):
            block = X[s:e]
        else:
            block = torch.from_numpy(np.array(X[s:e]))                    # a copy: memmaps are read-only
        yield block.to(device, torch.float32).contiguous()


def _check_n_components(n_components, n, d):
    if n_components is None:
        return min(n, d)
    if isinstance(n_components, (bool, np.bool_)) or not isinstance(n_components, (int, np.integer)):
        raise ValueError("n_components must be None or an int in [1, %d], got %r" % (min(n, d), n_components))
    if not 1 <= int(n_components) <= min(n, d):
        raise ValueError("n_components=%d must be between 1 and min(n_samples, n_features)=%d" % (n_components, min(n, d)))
    return int(n_components)


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
    n, d = _n_rows_dim(X)
    _check_n_components(n_components, max(n, 1), d)
    if n < 2:
        raise ValueError("a PCA fit needs at least 2 samples, got %d" % n)
    device = X.device if isinstance(X, torch.Tensor) and X.is_cuda else torch.device("cuda", torch.cuda.current_device())
    ops.require_gpu(device.index)
    with torch.cuda.device(device):                   # the library launches on the current device's current stream
        sums = torch.zeros(d, dtype=torch.float64, device=device)
        for x in _chunks(X, chunk_rows, device):
            ops.col_sums_f64(x, sums)
        sums_h = sums.cpu().numpy()
        if not np.all(np.isfinite(sums_h / n)):
            raise ValueError("Input contains NaN or infinity.")
        mean = sums / n
        gram = torch.zeros((d, d), dtype=torch.float64, device=device)
        for x in _chunks(X, chunk_rows, device):
            ops.gram_f64(x, mean, gram)
        gram_h = gram.cpu().numpy()
    return pca_from_gram(n, sums_h, gram_h, n_components)
