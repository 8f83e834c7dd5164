"""CPU checks of the AP-loss model (tests/aploss_model.py), the Python quantiser tables and the fp64 restatement of
the reference loss; each planted bug in the model is shown to leave a check; the kernels build without spills."""
import os
import re

import numpy as np
import pytest
import torch

import aploss_model as AM
import aploss_oracle as AO
from conftest import REPO


def test_tables_equal_reference(golden):
    from dirb200.loss import quantizer_table
    g = golden("aploss.npz")
    i = 0
    while "table.%d" % i in g:
        nq, lo, hi = g["table.%d.meta" % i]
        nq = int(nq)
        ref = g["table.%d" % i]
        assert quantizer_table(nq, lo, hi).numpy().view(np.uint32).tolist() == ref.view(np.uint32).tolist()
        w, b = AM.table(nq, lo, hi)
        assert np.array_equal(np.concatenate([w, b]).view(np.uint32), ref.view(np.uint32))
        wo, bo = AO.quantizer(nq, lo, hi)
        assert np.array_equal(torch.cat([wo, bo]).float().numpy().view(np.uint32), ref.view(np.uint32))
        i += 1
    assert i >= 8


def test_fmaf_single_rounding():
    r = np.random.RandomState(0)
    w = np.float32(-24.0 / 1.7)
    x = r.uniform(-2, 2, 20000).astype(np.float32)
    b = np.float32(13.123)
    from fractions import Fraction
    got = AM.fmaf(w, x, b)
    for xi, gi in zip(x[:400], got[:400]):
        exact = Fraction(float(w)) * Fraction(float(xi)) + Fraction(float(b))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda c: (abs(Fraction(float(c)) - exact), int(np.array(c).view(np.uint32)) & 1))
        assert gi == best


def _rand_hist(r, N, nq, mode, ties=False, empty=False):
    c = r.uniform(0, 30, (N, nq))
    cp = c * r.uniform(0, 1, (N, nq))
    if ties:
        cp[:, ::3] = 1.0
        c[:, 1::3] = 1.0
        cp[:, 1::3] = np.minimum(cp[:, 1::3], 1.0)
    if empty:
        c[:, :nq // 2] = 0
        cp[:, :nq // 2] = 0
    Np = np.maximum(cp.sum(1) + r.uniform(0, 2, N), 1e-3)
    h = np.zeros((N, 2 * nq + 1), np.int64)
    h[:, :nq] = np.rint(c * AM.FIX)
    h[:, nq:2 * nq] = np.rint(cp * AM.FIX)
    h[:, 2 * nq] = np.rint(Np * AM.FIX)
    return h


def _autograd_G(h, nq, mode):
    t = torch.from_numpy(h.astype(np.float64) / AM.FIX)
    c = t[:, :nq].clone().requires_grad_(True)
    cp = t[:, nq:2 * nq].clone().requires_grad_(True)
    ap = AO.rows(c, cp, t[:, 2 * nq:], mode)
    gc, gp = torch.autograd.grad(ap.sum(), (c, cp))
    return ap.detach().numpy(), np.concatenate([gc.numpy(), gp.numpy()], 1)


@pytest.mark.parametrize("mode", ["ap", "tap", "taps"])
@pytest.mark.parametrize("data", ["random", "ties", "empty"])
@pytest.mark.parametrize("nq", [2, 25, 100])
def test_coefficients_equal_autograd(mode, data, nq):
    h = _rand_hist(np.random.RandomState(nq), 40, nq, mode, ties=data == "ties", empty=data == "empty")
    ap, G, mag, Gm = AM.finalize(h, nq, mode)
    ap_r, G_r = _autograd_G(h, nq, mode)
    b_ap, b_G = AM.bounds(nq, mag, Gm)
    assert np.all(np.abs(ap - ap_r) <= b_ap)
    assert np.all(np.abs(G - G_r) <= b_G), np.max(np.abs(G - G_r) / np.maximum(b_G, 1e-300))


def _gold_model(g, name):
    nq, lo, hi = g[name + ".meta"]
    nq = int(nq)
    x, lab = g[name + ".x"], g[name + ".label"]
    mode = "tap" if name.startswith("tap") else "ap"
    return nq, lo, hi, x, lab, mode


@pytest.mark.parametrize("name", ["ap_nq2_0", "ap_nq25_-1", "ap_nq100_0", "tap", "ap_nopos", "ap_kinks",
                                  "tap_kinks"])
def test_oracle_and_model_against_goldens(golden, name):
    """The fp64 restatement and the model give the reference's per-row APs within its fp32 error (1e-4; M = 300)."""
    g = golden("aploss.npz")
    nq, lo, hi, x, lab, mode = _gold_model(g, name)
    ref = g[name + ".ap"]
    ora = AO.row_ap(torch.from_numpy(x).double(), torch.from_numpy(lab), nq, lo, hi, mode).numpy()
    w, b = AM.table(nq, lo, hi)
    mod, _, _, _ = AM.finalize(AM.histogram(x, lab, w, b, nq), nq, mode)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(ora), nan) and np.array_equal(np.isnan(mod), nan)
    assert np.all(np.abs(ora - ref)[~nan] <= 1e-4) and np.all(np.abs(mod - ref)[~nan] <= 1e-4)


def _model_grad(g, name, **bug):
    """x.grad of the golden case 'name' from the model: histogram -> G -> dx, with the case's objective."""
    nq, lo, hi, x, lab, mode = _gold_model(g, name)
    w, b = AM.table(nq, lo, hi)
    h = AM.histogram(x, lab, w, b, nq, round_fix=bug.get("round_fix", True))
    ap, G, _, _ = AM.finalize(h, nq, mode, eps=bug.get("eps"), rev_shift=bug.get("rev_shift", 0))
    ga = np.full(x.shape[0], -1.0 / x.shape[0], np.float32)
    dx, _ = AM.backward(x, lab, w, b, nq, G, ga, clamp_ge=bug.get("clamp_ge", True),
                        tie_split=bug.get("tie_split", True))
    return h, ap, dx


def test_model_gradient_matches_reference_on_kinks(golden):
    """On exact kinks (a = 16) the reference is exact too: same support and 1/2 factors, values within 1e-4."""
    g = golden("aploss.npz")
    for name in ("ap_kinks", "tap_kinks"):
        _, _, dx = _model_grad(g, name)
        ref = g[name + ".grad"]
        tiny = 1e-6 * np.max(np.abs(ref))        # the reference's fp32 cancellation leaves ~1e-12 where the sum is 0
        assert np.array_equal(np.abs(dx) > tiny, np.abs(ref) > tiny), name
        assert np.max(np.abs(dx - ref)) <= 1e-4 * np.max(np.abs(ref)), name


@pytest.mark.parametrize("bug", ["clamp_gt", "tie_one_branch", "truncate", "rev_cumsum", "no_eps"])
def test_planted_bugs_are_caught(golden, bug):
    g = golden("aploss.npz")
    if bug in ("clamp_gt", "tie_one_branch"):
        # the kink golden: support / values of x.grad differ from the reference's
        _, _, dx = _model_grad(g, "ap_kinks", **({"clamp_ge": False} if bug == "clamp_gt" else {"tie_split": False}))
        ref = g["ap_kinks.grad"]
        tiny = 1e-6 * np.max(np.abs(ref))
        assert (not np.array_equal(np.abs(dx) > tiny, np.abs(ref) > tiny)) or np.max(np.abs(dx - ref)) > 1e-4 * np.max(np.abs(ref))
    elif bug == "truncate":
        # the fixed-point bound against an exact sum: with the truncating model the histogram leaves it
        x, lab, exact = AM.fixed_point_case()
        w, b = AM.table(17, 0, 1)
        assert AM.fixed_point_error(AM.histogram(x, lab, w, b, 17), exact, x.size) <= 1
        assert AM.fixed_point_error(AM.histogram(x, lab, w, b, 17, round_fix=False), exact, x.size) > 1
    else:
        # the coefficient check against fp64 autograd (empty leading bins for eps)
        for nq in (25,):
            h = _rand_hist(np.random.RandomState(1), 40, nq, "ap", empty=True)
            ap, G, mag, Gm = AM.finalize(h, nq, "ap", **({"rev_shift": 1} if bug == "rev_cumsum" else {"eps": 0.0}))
            ap_r, G_r = _autograd_G(h, nq, "ap")
            b_ap, b_G = AM.bounds(nq, *AM.finalize(h, nq, "ap")[2:])
            ok = np.all(np.abs(ap - ap_r) <= b_ap) and np.all(np.abs(G - G_r) <= b_G)
            assert not ok


def test_new_kernels_do_not_spill():
    log = os.path.join(REPO, "deep-image-retrieval_b200", "build", "aploss.cu.log")
    if not os.path.exists(log):
        pytest.skip("no compiler log: the library was not built in this tree")
    text = open(log).read()
    blocks = re.findall(r"Compiling entry function '(\w+aploss_\w+)'.*?\n.*?\n(.*?)\n", text)
    assert len(blocks) == 3
    for name, stats in blocks:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in stats, (name, stats)


def test_python_surface_on_cpu():
    """Constructor arguments, assertions, measures() keys, and the triplet losses (pure torch)."""
    import dirtorch.loss as L
    for nq in (1, 101, 2.0):
        with pytest.raises(AssertionError):
            L.APLoss(nq=nq)
    with pytest.raises(AssertionError):
        L.APLoss(nq=10, min=1, max=1)
    t = L.TAPLoss(nq=10, simplified=True)
    assert t.nq == 10 and t.min == 0 and t.max == 1 and "table" not in t.state_dict()
    with pytest.raises(TypeError):
        L.APLoss()(torch.zeros(2, 3), torch.zeros(2, 3))
    a, p, n = (torch.randn(5, 8, dtype=torch.float64) for _ in range(3))
    for swap in (False, True):
        ref = torch.nn.functional.softplus(torch.nn.functional.pairwise_distance(a, p)
                                           - (torch.minimum(torch.nn.functional.pairwise_distance(a, n),
                                                            torch.nn.functional.pairwise_distance(p, n))
                                              if swap else torch.nn.functional.pairwise_distance(a, n))).mean()
        assert torch.allclose(L.TripletLogExpLoss(swap=swap)(a, p, n), ref)
    assert L.TripletMarginLoss(margin=0.5).eval_func(1.0, 2.0) == 0 and L.TripletMarginLoss(margin=0.5).eval_func(2.0, 1.0) == 1.5
    assert abs(L.TripletLogExpLoss().eval_func(1.0, 1.0) - np.log(2)) < 1e-12
    assert torch.allclose(L.sim_to_dist(torch.tensor([1.0, -1.0], dtype=torch.float64)),
                          torch.tensor([1 - 0.001 ** 0.5, 1 - 4.001 ** 0.5], dtype=torch.float64))
