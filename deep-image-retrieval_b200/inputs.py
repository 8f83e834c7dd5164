"""Descriptor inputs of the retrieval extensions: the device they run on, the rows they accept and the checks they
apply to their arguments.

Every entry point takes its rows as a CUDA tensor, a host tensor, a host array or memmap, or a ``DescriptorStore``;
``Rows`` reads any of them as fp32 device rows, whole or in chunks, so that host inputs larger than the device can be
streamed.
"""
from __future__ import annotations

import numpy as np
import torch

from .store import DescriptorStore

NORM_SLACK = 1e-3          # |norm - 1| that still counts as unit norm (the exact search's error bound allows it)


def device(device=None, X=None):
    """The device to run on: `device` when given, else the device of X when X is a CUDA tensor, else the current
    CUDA device."""
    if device is not None:
        return torch.device(device)
    if isinstance(X, torch.Tensor) and X.is_cuda:
        return X.device
    return torch.device("cuda", torch.cuda.current_device())


class Rows:
    """The (n, d) rows of X - a CUDA / host tensor, a host array / memmap / nested list, or a DescriptorStore.
    get(a, b, device): rows [a, b) as a contiguous fp32 tensor on `device`; a tensor that already is one comes back
    as itself, not as a copy."""

    def __init__(self, X, name="X"):
        if isinstance(X, DescriptorStore):
            self.n, self.d = len(X), X.dim
        else:
            if not isinstance(X, torch.Tensor) and not hasattr(X, "shape"):
                X = np.asarray(X, np.float32)
            if len(X.shape) != 2:
                raise ValueError("%s must be a 2-D array of descriptors (got shape %s)" % (name, tuple(X.shape)))
            self.n, self.d = int(X.shape[0]), int(X.shape[1])
        self.X = X

    def get(self, a, b, device):
        X = self.X
        if isinstance(X, DescriptorStore):
            return X.load_rows_to_device(a, b, device)[0]
        if isinstance(X, torch.Tensor):
            t = X if (a, b) == (0, self.n) else X[a:b]
        else:
            t = torch.from_numpy(np.require(X[a:b], np.float32, "CW"))     # a copy only when read-only: memmaps
        return t.to(device=device, dtype=torch.float32).contiguous()

    def chunks(self, chunk_rows, device):
        """The rows in order, chunk_rows at a time."""
        for a in range(0, self.n, chunk_rows):
            yield self.get(a, min(self.n, a + chunk_rows), device)


def rows(X, dev=None, name="X"):
    """All rows of X as a contiguous fp32 (N, D) tensor on dev (None: the current CUDA device)."""
    r = Rows(X, name)
    return r.get(0, r.n, device(dev))


def rows64(X):
    """All rows of X as fp32 on the current CUDA device, zero-padded to a multiple of 64 columns: the tensor-core
    search's layout, where zero columns change no score and no norm."""
    t = rows(X)
    pad = (-t.shape[1]) % 64
    return torch.nn.functional.pad(t, (0, pad)).contiguous() if pad else t


def check_int(v, name, lo=1, hi=None):
    """v as an int; ValueError unless it is an integer (not a bool) in [lo, hi] (hi None: no upper bound)."""
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo or (hi is not None and v > hi):
        raise ValueError("%s must be an integer %s (got %r)" % (name, ">= %d" % lo if hi is None else
                                                                "in [%d, %d]" % (lo, hi), v))
    return int(v)


def check_unit(x, name):
    """ValueError unless every row of x has |norm - 1| <= NORM_SLACK."""
    if x.shape[0]:
        worst = float((torch.linalg.vector_norm(x, dim=1) - 1.0).abs().max())
        if not worst <= NORM_SLACK:
            raise ValueError("%s rows must be unit-norm (largest |norm - 1| is %.4g)" % (name, worst))


def check_norm_at_most_1(x, name):
    """ValueError unless every row of x has norm <= 1 + NORM_SLACK: the exact search's error bound assumes it."""
    if x.shape[0]:
        worst = float(torch.linalg.vector_norm(x, dim=1).max())
        if worst > 1.0 + NORM_SLACK:
            raise ValueError("%s rows are not unit-norm (max norm %.4g): the exact-top-k error bound assumes |row| <= 1; "
                             "normalise them, or give eps16 = 1.2e-3*max|q|*max|row| + 2^-24*sqrt(D)*(max|q| + max|row|) "
                             "(entries below 65504; see ops.Index)" % (name, worst))
