"""fp64 restatement of the reference's APLoss / TAPLoss (dirtorch/loss.py), CPU torch, differentiable.

Kept apart from the numpy model of the kernels (tests/aploss_model.py), which it checks: it shares no code with it.
The quantiser is the reference's Conv1d (loss.py:29-41) with its fp32 parameters, evaluated in fp64; the AP and TAP
formulas are loss.py:50-55 and loss.py:104-119."""
import numpy as np
import torch


def quantizer(nq, lo, hi):
    """The reference's Conv1d weight and bias (loss.py:29-41): fp32 values, returned as fp64 tensors."""
    a = (nq - 1) / (hi - lo)
    w = torch.cat([torch.full((nq,), -a), torch.full((nq,), a)]).float()
    b = torch.cat([torch.from_numpy(a * lo + np.arange(nq, 0, -1)),
                   torch.from_numpy(np.arange(2 - nq, 2, 1) - a * lo)]).float()
    w[0] = w[-1] = 0
    b[0] = b[-1] = 1
    return w.double(), b.double()


def rows(c, cp, Np, mode):
    """Per-row AP from the bin sums c, cp and the positive count Np: mode 'ap' (loss.py:50-55), 'tap' or 'taps'
    (loss.py:104-119, simplified=False / True)."""
    if mode == "ap":
        prec = cp.cumsum(-1) / (1e-16 + c.cumsum(-1))
        return (prec * (cp / cp.sum(-1, keepdim=True))).sum(-1)
    C, Cp = c.cumsum(-1), cp.cumsum(-1)
    z = torch.zeros_like(C[:, :1])
    C1, Cp1 = torch.cat((z, C[:, :-1]), -1), torch.cat((z, Cp[:, :-1]), -1)
    if mode == "taps":
        aps = cp * (Cp1 + Cp + 1) / (C1 + C + 1) / Np
    else:
        eps = 1e-8
        ratio = (cp - 1).clamp(min=0) / ((c - 1).clamp(min=0) + eps)
        aps = cp * (c * ratio + (Cp1 + 1 - ratio * (C1 + 1)) * torch.log((C + 1) / (C1 + 1))) / (c + eps) / Np
    return aps.sum(-1)


def row_ap(x, label, nq, lo, hi, mode):
    """Per-row AP of scores x (N,M) fp64 (may require grad), labels {0,1} (loss.py:43-55 / 90-119)."""
    w, b = quantizer(nq, lo, hi)
    v = w.view(1, -1, 1) * x.unsqueeze(1) + b.view(1, -1, 1)
    q = torch.min(v[:, :nq], v[:, nq:]).clamp(min=0)
    lab = label.to(torch.float64)
    return rows(q.sum(-1), (q * lab.unsqueeze(1)).sum(-1), lab.sum(-1, keepdim=True), mode)
