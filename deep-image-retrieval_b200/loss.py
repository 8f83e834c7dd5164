"""Training losses of "Learning with Average Precision: Training Image Retrieval with a Listwise Loss" (Revaud et al.,
https://arxiv.org/abs/1906.07589), the reference's ``dirtorch/loss.py``.

``APLoss`` / ``TAPLoss`` (and their ``_dist`` variants) compute the per-row AP of quantised scores with two CUDA
kernels (csrc/aploss.cu): an exact fixed-point histogram of the 2nq soft bins and an fp64 finalisation that also
writes the gradient coefficients, then one elementwise backward pass.  Neither pass forms the N x 2nq x M tensor of
the reference's Conv1d quantiser, so memory stays at O(N M) bytes for dx and O(N nq) for the rest.

Differences from the reference:
- x must be an fp32 CUDA tensor (there is no CPU path).
- labels must be binary.  bool and uint8 labels are used as they are (uint8 is not checked: any non-zero value is
  a positive); other dtypes are checked once (one synchronisation) and non-binary values raise ``ValueError``.
- there is no ``quantizer`` submodule: the quantiser table is a non-persistent buffer built from (nq, min, max), so
  no state dict can make it disagree with the kernels.
- ``label.requires_grad`` raises; there is no double backward.
- the histograms are exact and the AP is finalised in fp64, so results are more accurate than the reference's fp32
  sums (and bit-identical from run to run).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

from . import ops


def quantizer_table(nq, min, max):
    """The 2nq weights and 2nq biases of the reference's quantiser Conv1d (loss.py:29-41), fp32, as one (4nq,) tensor.
    Lines 1..nq-1 fall from 1 at the bin's centre (slope -a), lines nq..2nq-2 rise to it (slope a); line 0 and line
    2nq-1 are the constant 1, which extends the end bins beyond [min, max]."""
    a = (nq - 1) / (max - min)
    w = np.empty(2 * nq, dtype=np.float32)
    w[:nq] = -a
    w[nq:] = a
    b = np.concatenate([a * min + np.arange(nq, 0, -1), np.arange(2 - nq, 2, 1) - a * min]).astype(np.float32)
    w[0] = w[-1] = 0
    b[0] = b[-1] = 1
    return torch.from_numpy(np.concatenate([w, b]))


def _binary_label(label):
    if label.requires_grad:
        raise ValueError("label must not require grad")
    if label.dtype == torch.bool:
        return label.contiguous().view(torch.uint8)
    if label.dtype == torch.uint8:
        return label.contiguous()
    if bool(((label != 0) & (label != 1)).any()):
        raise ValueError("labels must be binary (0 or 1)")
    return label.to(torch.uint8).contiguous()


class _RowAP(torch.autograd.Function):
    """(x, label) -> per-row AP, mode 'ap' / 'tap' / 'taps'."""

    @staticmethod
    def forward(ctx, x, label, table, nq, mode):
        _, G, ap = ops.aploss_forward(x, label, nq, table, mode)
        ctx.save_for_backward(x, label, table, G)
        ctx.nq = nq
        return ap

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_ap):
        x, label, table, G = ctx.saved_tensors
        dx = ops.aploss_backward(x, label, ctx.nq, table, G, grad_ap.float().contiguous())
        return dx, None, None, None, None


class APLoss(nn.Module):
    """Differentiable AP loss through quantisation (Revaud et al., 2019).

    Input x: (N, M) fp32 CUDA scores in [min, max]; label: (N, M) in {0, 1}.
    forward returns 1 - mAP (the mean over the N rows of their AP, optionally weighted by qw), or the per-row AP
    with ret='AP'."""
    _mode = "ap"
    _measure = "loss_ap"

    def __init__(self, nq=25, min=0, max=1):
        nn.Module.__init__(self)
        assert isinstance(nq, int) and 2 <= nq <= 100
        self.nq = nq
        self.min = min
        self.max = max
        gap = max - min
        assert gap > 0
        self.register_buffer("table", quantizer_table(nq, min, max), persistent=False)

    def row_ap(self, x, label):
        assert x.shape == label.shape  # N x M
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32):
            raise TypeError("x must be an fp32 CUDA tensor (there is no CPU path)")
        if not label.is_cuda or label.device != x.device:
            raise TypeError("label must be a CUDA tensor on the device of x")
        if self.table.device != x.device:
            self.table = self.table.to(x.device)
        return _RowAP.apply(x.contiguous(), _binary_label(label), self.table, self.nq, self._mode)

    def forward(self, x, label, qw=None, ret='1-mAP'):
        ap = self.row_ap(x, label)
        if ret == '1-mAP':
            if qw is not None:
                ap = ap * qw
            return 1 - ap.mean()
        elif ret == 'AP':
            assert qw is None
            return ap
        else:
            raise ValueError("Bad return type for APLoss(): %s" % str(ret))

    def measures(self, x, gt, loss=None):
        if loss is None:
            loss = self.forward(x, gt)
        return {self._measure: float(loss)}


class TAPLoss(APLoss):
    """Differentiable tie-aware AP loss through quantisation (Revaud et al., 2019); simplified=True uses the paper's
    simplified tie-aware precision.  Same inputs and outputs as APLoss."""

    def __init__(self, nq=25, min=0, max=1, simplified=False):
        APLoss.__init__(self, nq=nq, min=min, max=max)
        self.simplified = simplified
        self._mode = "taps" if simplified else "tap"
        self._measure = "loss_taps" if simplified else "loss_tap"


def sim_to_dist(scores):
    """Similarities of unit vectors -> 1 - (their Euclidean distance, with a 1e-3 margin under the square root)."""
    return 1 - torch.sqrt(2.001 - 2 * scores)


class APLoss_dist(APLoss):
    def forward(self, x, label, **kw):
        return APLoss.forward(self, sim_to_dist(x), label, **kw)


class TAPLoss_dist(TAPLoss):
    def forward(self, x, label, **kw):
        return TAPLoss.forward(self, sim_to_dist(x), label, **kw)


class TripletMarginLoss(nn.TripletMarginLoss):
    """torch's margin triplet loss; eval_func is the same hinge on two precomputed distances."""

    def eval_func(self, dp, dn):
        return max(0, dp - dn + self.margin)


class TripletLogExpLoss(nn.Module):
    """mean log(1 + exp(d(a, p) - d(a, n))) over (N, D) anchors, positives and negatives (Li et al., "Improving
    Pairwise Ranking for Multi-Label Image Classification").  swap=True uses min(d(a, n), d(p, n)) as the negative
    distance."""

    def __init__(self, p=2, eps=1e-6, swap=False):
        super().__init__()
        self.p, self.eps, self.swap = p, eps, swap

    def forward(self, anchor, positive, negative):
        assert anchor.size() == positive.size() == negative.size(), "anchor, positive and negative differ in size"
        assert anchor.dim() == 2, "Input must be a 2D matrix."
        d_p = F.pairwise_distance(anchor, positive, self.p, self.eps)
        d_n = F.pairwise_distance(anchor, negative, self.p, self.eps)
        if self.swap:
            d_n = torch.minimum(d_n, F.pairwise_distance(positive, negative, self.p, self.eps))
        return torch.log(1 + torch.exp(d_p - d_n)).mean()

    def eval_func(self, dp, dn):
        return np.log(1 + np.exp(dp - dn))
