"""GPU checks of the AP-loss kernels (csrc/aploss.cu) and of dirb200.loss.

- histograms equal the numpy model (tests/aploss_model.py) exactly;
- AP and G, teacher-forced from the kernel's own histogram, are within the model's fp64 bound; dx within its bound;
- against the unmodified reference (tests/golden/aploss.npz): losses, APs and x.grad within the reference's fp32 error;
- bit-identical reruns, and a row alone equals the same row in a 257-row batch;
- composition through x = D D^T against fp64 autograd of the reference formula; memory at N = M = 16384; errors."""
import numpy as np
import pytest
import torch

import aploss_model as AM
import aploss_oracle as AO

pytestmark = pytest.mark.gpu

RANGES = [(0, 1), (-1, 1), (-0.3, 2.5)]
SHAPES = [(N, M) for N in (1, 3, 257) for M in (1, 2, 31, 4097)]
WORST = {}


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest measured |delta| / bound:", {k: "%.3g" % v for k, v in sorted(WORST.items())})


def _table(nq, lo, hi):
    w, b = AM.table(nq, lo, hi)
    return w, b, torch.from_numpy(np.concatenate([w, b])).cuda()


def _fwd(x, lab, nq, lo, hi, mode):
    from dirb200 import ops
    w, b, t = _table(nq, lo, hi)
    h, G, ap = ops.aploss_forward(torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda(), nq, t, mode)
    return w, b, t, h.cpu().numpy(), G.cpu().numpy(), ap.cpu().numpy()


@pytest.mark.parametrize("kind", ["uniform", "outside", "concentrated", "kinks"])
@pytest.mark.parametrize("rng", RANGES)
@pytest.mark.parametrize("nq", [2, 3, 25, 100])
def test_histogram_exact(nq, rng, kind):
    lo, hi = rng
    for N, M in SHAPES:
        x, lab = AM.make_scores(1, N, M, nq, lo, hi, kind)
        w, b, _, h, _, _ = _fwd(x, lab, nq, lo, hi, "ap")
        ref = AM.histogram(x, lab, w, b, nq)
        assert np.array_equal(h, ref), (N, M, np.argwhere(h != ref)[:5])


def test_histogram_exact_long_rows():
    x, lab = AM.make_scores(2, 2, 1_000_003, 25, 0, 1, "outside")
    w, b, _, h, _, _ = _fwd(x, lab, 25, 0, 1, "ap")
    assert np.array_equal(h, AM.histogram(x, lab, w, b, 25))


def test_histogram_rounds_to_nearest():
    """Bin values with a fractional part of 3/4 in units of 2^-32 (exact sums known): the histogram is within half a
    unit per element of the exact sum, which a truncating conversion leaves."""
    x, lab, exact = AM.fixed_point_case()
    w, b, _, h, _, _ = _fwd(x, lab, 17, 0, 1, "ap")
    assert AM.fixed_point_error(h, exact, x.size) <= 1
    assert np.array_equal(h, AM.histogram(x, lab, w, b, 17))


def test_row_without_positive_is_nan_everywhere():
    """G of a row without positives is NaN; like the reference's conv backward, every element of dx is NaN, also where
    the active bin's slope is 0 (x above max, x on a bin's peak)."""
    import dirtorch.loss as L
    x = torch.tensor([[1.5, 1.0, 0.5, 0.25, -0.5, 0.3], [1.5, 1.0, 0.5, 0.25, -0.5, 0.3]], device="cuda",
                     requires_grad=True)
    lab = torch.tensor([[0, 0, 0, 0, 0, 0], [1, 0, 1, 0, 0, 1]], device="cuda", dtype=torch.bool)
    ap = L.APLoss(nq=17)(x, lab, ret='AP')
    ap.sum().backward()
    assert torch.isnan(ap[0]) and torch.isfinite(ap[1])
    assert torch.isnan(x.grad[0]).all() and torch.isfinite(x.grad[1]).all()


@pytest.mark.parametrize("mode", ["ap", "tap", "taps"])
@pytest.mark.parametrize("nq", [2, 25, 100])
@pytest.mark.parametrize("kind", ["uniform", "outside", "concentrated", "kinks"])
def test_ap_g_dx_within_bounds(mode, nq, kind):
    from dirb200 import ops
    x, lab = AM.make_scores(3, 257, 999, nq, 0, 1, kind)
    w, b, t, h, G, ap = _fwd(x, lab, nq, 0, 1, mode)
    ap_m, G_m, mag, Gm = AM.finalize(h, nq, mode)
    b_ap, b_G = AM.bounds(nq, mag, Gm)
    b_ap = b_ap + np.abs(ap_m) * 2.0 ** -24            # the fp32 rounding of the AP
    d_ap = np.abs(ap.astype(np.float64) - ap_m)
    assert np.all(d_ap <= b_ap), np.max(d_ap / b_ap)
    _note("ap " + mode, np.max(d_ap / b_ap))
    d_G = np.abs(G - G_m)
    assert np.all(d_G <= b_G), np.max(d_G / np.maximum(b_G, 1e-300))
    _note("G " + mode, np.max(np.where(b_G > 0, d_G / np.maximum(b_G, 1e-300), 0)))
    g = np.random.RandomState(4).standard_normal(257).astype(np.float32)
    dx = ops.aploss_backward(torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda(), nq, t,
                             torch.from_numpy(G).cuda(), torch.from_numpy(g).cuda()).cpu().numpy()
    dx_m, dmag = AM.backward(x, lab, w, b, nq, G, g)
    bound = np.abs(dx_m).astype(np.float64) * 2.0 ** -23 + 2 * AM.gamma(8) * dmag + 1e-300
    d = np.abs(dx.astype(np.float64) - dx_m)
    assert np.all(d <= bound), np.max(d / bound)
    _note("dx " + mode, np.max(d / bound))


def _near_kink(x, nq, lo, hi, tol=1e-5):
    """Elements whose quantiser value or min branch is within tol of a kink, where the reference's CPU rounding of v
    (a product and a sum, not an fma) can take the other side."""
    w, b = AM.table(nq, lo, hi)
    v = w.astype(np.float64)[None, :, None] * x.astype(np.float64)[:, None, :] + b.astype(np.float64)[None, :, None]
    lo_, hi_ = v[:, :nq], v[:, nq:]
    m = np.minimum(lo_, hi_)
    near = (np.abs(m) < tol) | ((np.abs(lo_ - hi_) < tol) & (m > -tol))
    return near.any(1)


def _straddles_one(x, lab, nq, lo, hi):
    """TAP rows whose fp32 bin sums c or cp lie within 1e-3 of 1, the kink of relu(c - 1)."""
    w, b = AM.table(nq, lo, hi)
    h = AM.histogram(x, lab, w, b, nq).astype(np.float64) / AM.FIX
    return (np.abs(h[:, :2 * nq] - 1) < 1e-3).any(1)


GOLD_CASES = ["ap_nq2_0", "ap_nq2_-1", "ap_nq25_0", "ap_nq25_-1", "ap_nq100_0", "ap_nq100_-1", "tap", "taps",
              "ap_qw", "ap_ret", "ap_dist", "tap_dist", "ap_nopos", "ap_kinks", "tap_kinks"]


@pytest.mark.parametrize("name", GOLD_CASES)
def test_against_reference_goldens(golden, name):
    """The reference sums M fp32 products per bin (M = 300), so its bin sums, APs and x.grad carry a relative error of
    about M * 2^-24 = 1.8e-5; the bar is 1e-4 on the losses and APs and 1e-4 * max |x.grad| of the case on x.grad, with
    elements within 1e-5 of a kink, and TAP rows whose sums straddle 1, excluded (named in the assertion messages)."""
    import dirtorch.loss as L
    g = golden("aploss.npz")
    nq, lo, hi = g[name + ".meta"]
    nq = int(nq)
    cls = {"tap": L.TAPLoss, "taps": L.TAPLoss, "ap_dist": L.APLoss_dist, "tap_dist": L.TAPLoss_dist,
           "tap_kinks": L.TAPLoss}.get(name, L.APLoss)
    kw = {"simplified": True} if name == "taps" else {}
    mod = cls(nq=nq, min=lo, max=hi, **kw)
    x = torch.from_numpy(g[name + ".x"]).cuda().requires_grad_(True)
    lab = torch.from_numpy(g[name + ".label"]).cuda()
    ap = mod(x, lab, ret='AP').detach().cpu().numpy()
    if name + ".weights" in g:
        loss = (mod(x, lab, ret='AP') * torch.from_numpy(g[name + ".weights"]).cuda()).sum()
    else:
        qw = torch.from_numpy(g[name + ".qw"]).cuda() if name + ".qw" in g else None
        loss = mod(x, lab, qw=qw)
    loss.backward()
    grad = x.grad.cpu().numpy()
    ref_ap, ref_grad = g[name + ".ap"], g[name + ".grad"]
    nan_rows = np.isnan(ref_ap)
    assert np.array_equal(np.isnan(ap), nan_rows)
    if name == "ap_nopos":
        assert nan_rows[2] and nan_rows.sum() == 1 and np.isnan(grad[2]).all()
    else:
        assert abs(float(loss) - float(g[name + ".loss"])) <= 1e-4
    assert np.all(np.abs(ap - ref_ap)[~nan_rows] <= 1e-4)
    xin = g[name + ".x"]
    if "dist" in name:
        xin = (1 - np.sqrt(2.001 - 2 * xin.astype(np.float64))).astype(np.float32)
    exact = "kinks" in name                      # a = 16: every table value and v is exact in fp32
    skip = np.zeros(xin.shape, bool) if exact else _near_kink(xin, nq, lo, hi)
    if name.startswith("tap"):
        skip |= _straddles_one(xin, g[name + ".label"], nq, lo, hi)[:, None]
    skip |= nan_rows[:, None]
    tol = 1e-4 * np.nanmax(np.abs(ref_grad))
    bad = (np.abs(grad - ref_grad) > tol) & ~skip
    assert not bad.any(), ("elements off", np.argwhere(bad)[:5], "excluded", np.argwhere(skip & ~nan_rows[:, None])[:5])
    if exact:
        # the support and the 1/2 factors of the subgradient are the reference's
        tiny = 1e-6 * np.max(np.abs(ref_grad))   # the reference's fp32 cancellation leaves ~1e-12 where the sum is 0
        assert np.array_equal(np.abs(grad) > tiny, np.abs(ref_grad) > tiny)


def test_kink_gradient_example():
    """x = 0.5 with nq = 17 on [0, 1]: bins 7, 8, 9 take part (8 at its peak with slope 0, 7 and 9 at exactly 0)."""
    import dirtorch.loss as L
    x = torch.tensor([[0.5, 0.1, 0.9, 0.3]], device="cuda", requires_grad=True)
    lab = torch.tensor([[1, 0, 1, 0]], device="cuda", dtype=torch.bool)
    loss = L.APLoss(nq=17)(x, lab)
    loss.backward()
    x64 = x.detach().cpu().double().requires_grad_(True)
    ref = 1 - AO.row_ap(x64, lab.cpu(), 17, 0, 1, "ap").mean()
    ref.backward()
    assert torch.allclose(x.grad.cpu().double(), x64.grad, rtol=1e-6, atol=1e-7), (x.grad, x64.grad)


@pytest.mark.parametrize("mode", ["ap", "tap", "taps"])
def test_determinism_and_batch_invariance(mode):
    from dirb200 import ops
    nq = 25
    x, lab = AM.make_scores(5, 257, 5000, nq, 0, 1, "outside")
    _, _, t = _table(nq, 0, 1)
    xt, lt = torch.from_numpy(x).cuda(), torch.from_numpy(lab).cuda()
    g = torch.ones(257, device="cuda")
    runs = []
    for _ in range(2):
        h, G, ap = ops.aploss_forward(xt, lt, nq, t, mode)
        dx = ops.aploss_backward(xt, lt, nq, t, G, g)
        runs.append((h.cpu(), G.cpu(), ap.cpu(), dx.cpu()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    for r in (0, 128, 256):
        h1, G1, ap1 = ops.aploss_forward(xt[r:r + 1].contiguous(), lt[r:r + 1].contiguous(), nq, t, mode)
        dx1 = ops.aploss_backward(xt[r:r + 1].contiguous(), lt[r:r + 1].contiguous(), nq, t, G1, g[:1].contiguous())
        assert torch.equal(h1.cpu()[0], runs[0][0][r]) and torch.equal(G1.cpu()[0], runs[0][1][r])
        assert torch.equal(ap1.cpu()[0], runs[0][2][r]) and torch.equal(dx1.cpu()[0], runs[0][3][r])


@pytest.mark.parametrize("variant", ["ap_qw", "ap_ret", "ap_dist", "tap_dist", "taps"])
def test_composition_through_gram(variant):
    """x = D D^T with D requiring grad.  D.grad is compared with CPU fp64 autograd of the reference formula on the same
    D: the scores differ by fp32 rounding (|x| <= 1, ~1e-7), which moves the loss by ~1e-6 and, for the few elements
    within 1e-7 of a kink, flips a subgradient; the bar is 1e-3 relative L2 on D.grad and 1e-5 on the loss."""
    import dirtorch.loss as L
    torch.backends.cuda.matmul.allow_tf32 = False
    r = np.random.RandomState(6)
    D = r.standard_normal((96, 32))
    D *= 0.9 / np.linalg.norm(D, axis=1, keepdims=True)   # the diagonal at 0.81, not on the kink at max = 1
    cls_id = r.randint(0, 6, 96)
    lab = torch.from_numpy(cls_id[:, None] == cls_id[None, :])
    lo, hi = (-1, 1)
    mode = {"tap_dist": "tap", "taps": "taps"}.get(variant, "ap")
    mod = {"ap_qw": L.APLoss, "ap_ret": L.APLoss, "ap_dist": L.APLoss_dist, "tap_dist": L.TAPLoss_dist,
           "taps": L.TAPLoss}[variant](nq=25, min=lo, max=hi, **({"simplified": True} if variant == "taps" else {}))
    qw = torch.from_numpy(r.uniform(0.5, 2, 96))
    wv = torch.from_numpy(r.standard_normal(96))
    Dg = torch.from_numpy(D).float().cuda().requires_grad_(True)
    D64 = torch.from_numpy(D).requires_grad_(True)

    def objective(x, ap_fn, qw_, wv_):
        if variant == "ap_ret":
            return (ap_fn(x) * wv_).sum()
        ap = ap_fn(x)
        return 1 - (ap * qw_).mean() if variant == "ap_qw" else 1 - ap.mean()

    x = Dg @ Dg.T
    if variant == "ap_ret":
        loss = (mod(x, lab.cuda(), ret='AP') * wv.float().cuda()).sum()
    elif variant == "ap_qw":
        loss = mod(x, lab.cuda(), qw=qw.float().cuda())
    else:
        loss = mod(x, lab.cuda())
    loss.backward()
    x64 = D64 @ D64.T
    if "dist" in variant:
        x64 = 1 - torch.sqrt(2.001 - 2 * x64)
    ref = objective(x64, lambda s: AO.row_ap(s, lab, 25, lo, hi, mode), qw, wv)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5
    err = float(torch.linalg.norm(Dg.grad.cpu().double() - D64.grad) / torch.linalg.norm(D64.grad))
    assert err <= 1e-3, err


def test_memory_at_16384():
    """forward + backward at N = M = 16384, nq = 100: the peak allocation above the inputs is dx + hist + G plus
    16 MiB (the per-row AP, its gradient and allocator rounding).  The reference formulation would hold
    N * 2nq * M * 4 bytes = 215 GB for the Conv1d output alone."""
    import dirtorch.loss as L
    N = M = 16384
    nq = 100
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((N, M), device="cuda", generator=g).requires_grad_(True)
    lab = torch.rand((N, M), device="cuda", generator=g) < 0.01
    mod = L.APLoss(nq=nq)
    mod.table = mod.table.cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = mod(x, lab)
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    allowed = N * M * 4 + N * (2 * nq + 1) * 8 + N * 2 * nq * 8 + (16 << 20)
    assert peak <= allowed, (peak, allowed)
    assert torch.isfinite(loss) and torch.isfinite(x.grad).all()


def test_errors():
    import dirtorch.loss as L
    mod = L.APLoss(nq=25)
    x = torch.rand(4, 10, device="cuda")
    lab = torch.zeros(4, 10, device="cuda", dtype=torch.bool)
    with pytest.raises(TypeError):
        mod(x.cpu(), lab.cpu())
    with pytest.raises(TypeError):
        mod(x.half(), lab)
    with pytest.raises(ValueError):
        mod(x, torch.full((4, 10), 0.5, device="cuda"))
    with pytest.raises(ValueError):
        mod(x, torch.zeros(4, 10, device="cuda").requires_grad_(True))
    for nq in (1, 101):
        with pytest.raises(AssertionError):
            L.APLoss(nq=nq)
    with pytest.raises(AssertionError):
        mod(x, lab[:, :5])
    float_lab = (torch.rand(4, 10, device="cuda") < 0.3).float()
    float_lab[:, 0] = 1
    assert torch.equal(mod(x, float_lab, ret='AP'), mod(x, float_lab.bool(), ret='AP'))
