#!/usr/bin/env python
"""Generate tests/golden/aploss.npz by running the UNMODIFIED reference loss (dirtorch/loss.py) on the CPU.

    python tests/golden/make_golden_aploss.py

Like make_golden.py it imports naver/deep-image-retrieval from /root/reference (read-only, nothing is copied).  The
seeded inputs come from tests/aploss_model.py (synthdata's generators) and are stored with the outputs, since they are
small.  Stored per case <name>: x, label, nq, lo, hi, loss, ap (per-row, ret='AP') and grad (x.grad of the case's
objective); per quantiser: table_<nq>_<i> (the reference's fp32 Conv1d weight and bias)."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, REF)
sys.path.append(os.path.join(REPO, "tests"))

import torch  # noqa: E402

import dirtorch.loss as L  # noqa: E402  (the reference)
import aploss_model as AM  # noqa: E402

assert L.__file__.startswith(REF), L.__file__

TABLES = [(2, 0, 1), (3, 0, 1), (17, 0, 1), (25, 0, 1), (100, 0, 1), (25, -1, 1), (100, -1, 1), (7, -0.3, 2.5)]


def case(out, name, cls, nq, lo, hi, x, label, objective="mean", qw=None, **kw):
    torch.manual_seed(0)
    loss_mod = cls(nq=nq, min=lo, max=hi, **kw)
    xt = torch.from_numpy(x).requires_grad_(True)
    lt = torch.from_numpy(label)
    with torch.no_grad():
        ap = loss_mod(xt, lt, ret='AP')
    if objective == "mean":
        loss = loss_mod(xt, lt, qw=None if qw is None else torch.from_numpy(qw))
        loss.backward()
    else:                                   # ret='AP' backpropagated through a seeded weight vector
        wv = AM.synth._rs(7, name).standard_normal(x.shape[0])
        loss = (loss_mod(xt, lt, ret='AP') * torch.from_numpy(wv).float()).sum()
        loss.backward()
        out[name + ".weights"] = wv.astype(np.float32)
    out[name + ".x"] = x
    out[name + ".label"] = label
    out[name + ".meta"] = np.array([nq, lo, hi], np.float64)
    out[name + ".loss"] = np.float32(loss.item())
    out[name + ".ap"] = ap.numpy()
    out[name + ".grad"] = xt.grad.numpy()
    if qw is not None:
        out[name + ".qw"] = qw


def main():
    out = {}
    for i, (nq, lo, hi) in enumerate(TABLES):
        q = L.APLoss(nq=nq, min=lo, max=hi).quantizer
        out["table.%d" % i] = np.concatenate([q.weight.detach().view(-1).numpy(), q.bias.detach().numpy()])
        out["table.%d.meta" % i] = np.array([nq, lo, hi], np.float64)
    for nq in (2, 25, 100):
        for lo, hi in ((0, 1), (-1, 1)):
            x, lab = AM.make_scores(11, 6, 300, nq, lo, hi, "outside" if nq == 25 else "uniform")
            case(out, "ap_nq%d_%g" % (nq, lo), L.APLoss, nq, lo, hi, x, lab)
    x, lab = AM.make_scores(12, 6, 300, 25, 0, 1, "uniform")
    case(out, "tap", L.TAPLoss, 25, 0, 1, x, lab)
    case(out, "taps", L.TAPLoss, 25, 0, 1, x, lab, simplified=True)
    qw = AM.synth._rs(13, "qw").uniform(0.5, 2, 6).astype(np.float32)
    case(out, "ap_qw", L.APLoss, 25, 0, 1, x, lab, qw=qw)
    case(out, "ap_ret", L.APLoss, 25, 0, 1, x, lab, objective="AP")
    s, lab2 = AM.make_scores(14, 6, 300, 25, -1, 1, "uniform")
    case(out, "ap_dist", L.APLoss_dist, 25, -1, 1, s, lab2)
    case(out, "tap_dist", L.TAPLoss_dist, 25, -1, 1, s, lab2)
    lab3 = lab.copy()
    lab3[2] = 0                             # a row without positives: NaN AP
    case(out, "ap_nopos", L.APLoss, 25, 0, 1, x, lab3, objective="AP")
    xk, labk = AM.make_scores(15, 6, 300, 17, 0, 1, "kinks")
    case(out, "ap_kinks", L.APLoss, 17, 0, 1, xk, labk)
    case(out, "tap_kinks", L.TAPLoss, 17, 0, 1, xk, labk)
    path = os.path.join(HERE, "aploss.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
