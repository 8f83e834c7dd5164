"""The kernels between the layer4 map and the index, element by element against the fp64 references and bounds of
tests/post_model.py, each teacher-forced from the GPU's own input: the head phase by phase (fused and per phase), center
bias, both whitening paths and the L2 after them, scale pooling, row L2, the fp16 copies, alpha-QE and the dense exact
scores, at the shapes and data where such kernels break.  Needs an H100: -m gpu.

Each check prints a line ``POST <kernel> <case>: ratio r`` (the largest |gpu - ref| / bound) and, for whiten_tc,
``kappa r`` (the largest accumulation ratio, which sets post_model.KAPPA_W)."""
import ctypes as C

import numpy as np
import pytest
import torch

import post_model as PM

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _ops():
    from dirb200 import ops
    ops.require_gpu(0)
    return ops


def _ok(kernel, case, c, extra=""):
    print("POST %s %s: ratio %.4f%s" % (kernel, case, c.ratio, extra))
    assert c.ok, "%s %s: %d / %d elements outside the bound; %s" % (kernel, case, c.n_fail, c.n, c.worst)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# --------------------------------------------------------------------------- head
def _head_run(feat, pooling, p, eps, nf, fc_w, fc_b, fused):
    """dirb200_head_pool_fc_l2 with a workspace owned here -> partial, g, y read at the library's offsets."""
    from dirb200 import lib, ops
    B, H, W, Cc = feat.shape
    O = fc_w.shape[0] if fc_w is not None else Cc
    lay = PM.head_layout(B, H * W, Cc, O)
    assert lay["total"] == lib.raw("dirb200_head_workspace_floats")(B, H * W, Cc, O)
    ws = torch.full((lay["total"],), float("nan"), dtype=torch.float32, device=DEV)
    ws[-32:] = 0
    desc = torch.empty((B, O), dtype=torch.float32, device=DEV)
    d16 = torch.empty((B, O), dtype=torch.float16, device=DEV)
    saved = ops.get_global_option("head_fused")
    try:
        ops.set_global_option("head_fused", fused)
        lib.call("dirb200_head_pool_fc_l2", ops._ptr(feat), B, H * W, Cc, ops.POOLING[pooling], float(p), float(eps), int(nf),
                 ops._ptr(fc_w), ops._ptr(fc_b), O, ops._ptr(ws), ops._ptr(desc), ops._ptr(d16), ops._stream())
        torch.cuda.synchronize()
    finally:
        ops.set_global_option("head_fused", saved)
    S = lay["S"]
    return dict(partial=ws[:B * S * Cc].view(B, S, Cc), g=ws[lay["g"]:lay["g"] + B * Cc].view(B, Cc),
                y=ws[lay["y"]:lay["y"] + B * O].view(B, O) if fc_w is not None else None, desc=desc, desc16=d16)


def _feat(B, H, W, Cc, data, seed):
    r = np.random.RandomState(seed)
    x = np.abs(r.standard_normal((B, H, W, Cc))).astype(np.float32)
    if data == "edges":
        x[0, ..., : min(Cc, 9)] = 0                                     # whole zero channels: clamp to eps
        x[..., 9:17] = 0
        x.reshape(B, -1, Cc)[:, ::3, 17:40] = r.uniform(0, 6e-5, x.reshape(B, -1, Cc)[:, ::3, 17:40].shape)   # fp16 subnormals
        x.reshape(-1)[::101] = 0
    if data == "large":
        x = (x / x.max() * 65504.0).astype(np.float32)
        x.reshape(-1)[::7] = 65504.0
    return _t(x.astype(np.float16))


HEAD_CASES = [
    # B, H, W, C, out_dim (None = without_fc), pooling, p, norm_features, data
    (1, 1, 1, 2048, 2048, "gem", 3.0, False, "normal"),
    (7, 7, 9, 2048, 128, "gem", 3.0, False, "edges"),
    (8, 8, 8, 512, 1000, "gem", 2.5, True, "normal"),
    (9, 5, 13, 520, 520, "gem", 3.0000002, False, "edges"),
    (64, 4, 16, 2048, 2048, "gem", 3.0, False, "normal"),
    (2, 1, 63, 2048, 3072, "avg", 3.0, False, "edges"),
    (3, 5, 13, 2048, None, "max", 3.0, False, "edges"),
    (2, 8, 16, 520, 1000, "max", 3.0, True, "normal"),
    (1, 32, 32, 2048, 2048, "gem", 3.0, False, "edges"),
    (2, 64, 64, 2048, 2048, "gem", 2.5, False, "normal"),
    (1, 37, 29, 512, None, "gem", 3.0000002, True, "normal"),
    (9, 16, 64, 512, 3072, "avg", 3.0, False, "normal"),
    (2, 13, 5, 2048, 2048, "gem", 3.0, False, "large"),
    (8, 9, 15, 2048, 7, "gem", 3.0, False, "normal"),
]


@pytest.mark.parametrize("fused", [1, 0], ids=["fused", "phases"])
@pytest.mark.parametrize("case", HEAD_CASES, ids=lambda c: "%dx%dx%dx%d-%s-%s-%g%s-%s" % (
    c[0], c[1], c[2], c[3], c[4], c[5], c[6], "-nf" if c[7] else "", c[8]))
def test_head_every_phase(case, fused):
    """Partial sums (split counts 1..16, per not dividing HW, the c0 < C guard at C = 520), the pooled g, FC + bias
    (batch groups of 8, out_dim not a multiple of 8), the L2, desc16 == desc.half(), and the end-to-end bound from the
    fp16 map; fused kernel and phase kernels."""
    _ops()
    B, H, W, Cc, O, pooling, p, nf, data = case
    feat = _feat(B, H, W, Cc, data, seed=B * 131 + H * W + Cc)
    r = np.random.RandomState(Cc + (O or 0))
    fc_w = fc_b = None
    if O is not None:
        fc_w = _t((r.standard_normal((O, Cc)) / np.sqrt(Cc)).astype(np.float32))
        fc_b = _t((0.01 * r.standard_normal(O)).astype(np.float32))
    out = _head_run(feat, pooling, p, 1e-6, nf, fc_w, fc_b, fused)
    name = "%s/%s" % (pooling, "fused" if fused else "phases")
    f3 = feat.reshape(B, H * W, Cc)
    P, eP = PM.head_partial_ref(f3, pooling, p, 1e-6)
    _ok("head_partial", name, PM.check("partial", out["partial"], P, eP))
    if not nf:
        g, eg = PM.head_pool_final_ref(out["partial"], H * W, pooling, p, False)
        _ok("head_pool", name, PM.check("g", out["g"], g, eg))
    else:                                        # g is normalised in place: check the composition from the partials
        g, eg = PM.head_pool_final_ref(out["partial"], H * W, pooling, p, True)
        _ok("head_pool_l2", name, PM.check("g", out["g"], g, eg))
    pre = out["g"]
    if fc_w is not None:
        y, ey = PM.head_fc_ref(out["g"], fc_w, fc_b)
        _ok("head_fc", name, PM.check("y", out["y"], y, ey))
        pre = out["y"]
    d, ed = PM.l2_ref(pre, eps=1e-12)
    _ok("head_l2", name, PM.check("desc", out["desc"], d, ed))
    assert PM.half_bits_equal(out["desc16"], out["desc"])
    ref, bound = PM.head_e2e(f3, pooling, p, 1e-6, nf, fc_w, fc_b)
    _ok("head_e2e", name, PM.check("e2e", out["desc"], ref, bound))


# --------------------------------------------------------------------------- center bias
@pytest.mark.parametrize("shape", [(2, 7, 7, 64), (1, 7, 12, 2048), (3, 23, 17, 512), (1, 1, 1, 8), (1, 1, 5, 16), (2, 32, 32, 2048)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("b", [0.5, 1.0, 3.7])
def test_center_bias(shape, b):
    ops = _ops()
    r = np.random.RandomState(sum(shape))
    x = np.abs(r.standard_normal(shape)).astype(np.float32) * 8
    x.reshape(-1)[::5] = 65504.0 / (1 + b) * 0.99
    x.reshape(-1)[::11] = 3e-7
    x16 = _t(x.astype(np.float16))
    y = ops.center_bias(x16.clone(), b)
    torch.cuda.synchronize()
    _ok("center_bias", "%s b%g" % ("x".join(map(str, shape)), b), PM.center_bias_check("cb", y, x16, b))
    assert torch.equal(ops.center_bias(x16.clone(), 0.0), x16)


# --------------------------------------------------------------------------- whitening
def _whiten_data(N, D, Dout, data, seed):
    r = np.random.RandomState(seed)
    comp = (r.standard_normal((Dout, D)) / np.sqrt(D)).astype(np.float32)
    mean = (0.05 * r.standard_normal(D)).astype(np.float32)
    cs = r.uniform(0.3, 5.0, Dout).astype(np.float32)
    X = r.standard_normal((N, D)) / np.sqrt(D)
    if data == "clustered":
        X = mean + 1e-3 * X / np.linalg.norm(X, axis=1, keepdims=True)
    elif data == "mixed":
        X = X * np.logspace(-3, np.log10(300.0), N)[:, None]
    elif data == "edges":
        X[0] = mean
        comp[:, 1] = r.standard_normal(Dout) * 2.0 ** -20
        X[:, 2] *= 2.0 ** -20
    else:
        X = X + mean
    return X.astype(np.float32), comp, mean, cs


WHITEN_CASES = [
    # N, D, Dout, data, mean, colscale
    (1, 48, 7, "normal", True, True),
    (10, 48, 64, "normal", True, False),
    (55, 2048, 1000, "normal", True, True),
    (63, 512, 129, "edges", True, True),
    (64, 2048, 1, "normal", True, True),
    (65, 512, 127, "clustered", True, True),
    (127, 2048, 128, "mixed", True, True),
    (128, 512, 2048, "normal", False, False),
    (129, 2048, 129, "edges", True, True),
    (5063, 2048, 2048, "normal", True, True),
    (1000, 2048, 7, "clustered", True, False),
    (300, 48, 1000, "mixed", True, True),
    (777, 512, 1000, "mixed", False, True),
]


@pytest.mark.parametrize("case", WHITEN_CASES, ids=lambda c: "%dx%dx%d-%s%s%s" % (
    c[0], c[1], c[2], c[3], "" if c[4] else "-nomean", "" if c[5] else "-nocs"))
def test_whiten_both_paths(case):
    """SIMT path (N < 64 or D % 64 != 0) to its gamma_D bound, tensor-core path to KAPPA_W; then the L2 (eps 0) from
    the un-normalised output, and y16 == y.half() with and without the L2."""
    ops = _ops()
    N, D, Dout, data, use_mean, use_cs = case
    X, comp, mean, cs = _whiten_data(N, D, Dout, data, seed=N + D + Dout)
    x, c = _t(X), _t(comp)
    m, s = (_t(mean) if use_mean else None), (_t(cs) if use_cs else None)
    y, y16 = ops.whiten(x, c, m, s, l2norm=False, want_f16=True)
    yl, yl16 = ops.whiten(x, c, m, s, l2norm=True, want_f16=True)
    torch.cuda.synchronize()
    name = "%dx%dx%d-%s" % (N, D, Dout, data)
    if D % 64 == 0 and N >= 64:
        ref, bound, acc = PM.whiten_tc_ref(x, c, m, s)
        d = (y.double() - ref).abs() - PM.U * y.double().abs()
        kappa = float((d / torch.where(acc > 0, acc, torch.ones_like(acc))).max())
        _ok("whiten_tc", name, PM.check("y", y, ref, bound), ", kappa %.4f" % kappa)
    else:
        ref, bound = PM.whiten_simt_ref(x, c, m, s)
        _ok("whiten_simt", name, PM.check("y", y, ref, bound))
    assert PM.half_bits_equal(y16, y)
    lref, lbound = PM.l2_ref(y, eps=0.0)
    _ok("whiten_l2", name, PM.check("yl", yl, lref, lbound))
    assert PM.half_bits_equal(yl16, yl)


def test_whiten_tc_split_error_stays_inside_its_bound():
    """The hi/lo split's own error against the fp32 operands: within split_error_bound, so the tensor-core bound plus
    it bounds the whitening against the exact product of the fp32 inputs."""
    _ops()
    X, comp, mean, cs = _whiten_data(500, 2048, 256, "mixed", seed=3)
    x, c, m = _t(X), _t(comp), _t(mean)
    hx, lx, hc, lc, cse = PM.whiten_tc_parts(x, c, m)
    exact = PM.centred(x, m).double() @ c.double().T
    approx = (hx @ lc.T + lx @ hc.T + hx @ hc.T) * cse
    assert bool(((approx - exact).abs() <= PM.split_error_bound(x, c, m)).all())


# --------------------------------------------------------------------------- scale pooling
@pytest.mark.parametrize("S", [1, 2, 3, 5])
@pytest.mark.parametrize("N,D", [(1, 1), (1000, 7), (1, 256), (1000, 257), (1, 2048)], ids=lambda v: str(v))
@pytest.mark.parametrize("pooling,gemp", [("mean", 3.0), ("gem", 3.0), ("gem", 2.5)], ids=["mean", "gem3", "gem2.5"])
def test_pool_scales(S, N, D, pooling, gemp):
    """Both signs, exact zeros, |v| < 1e-6 (the clamp), chains that cancel (zero crossings of the mean); then the L2."""
    ops = _ops()
    r = np.random.RandomState(S * 1000 + D)
    xs = [r.standard_normal((N, D)).astype(np.float32) for _ in range(S)]
    if S > 1:
        xs[1][:, ::3] = -xs[0][:, ::3] * np.float32(1 + 1e-6)
    xs[0][:, 1::5] = 0
    xs[-1][:, 2::7] = 3e-7 * np.sign(r.standard_normal(xs[-1][:, 2::7].shape))
    t = [_t(v) for v in xs]
    out = ops.pool_scales(t, pooling, gemp, l2=False)
    outl = ops.pool_scales(t, pooling, gemp, l2=True)
    torch.cuda.synchronize()
    ref, bound = PM.pool_scales_ref(t, pooling, gemp)
    name = "S%d %dx%d %s%g" % (S, N, D, pooling, gemp)
    _ok("pool_scales", name, PM.check("pool", out, ref, bound))
    lref, lbound = PM.l2_ref(out, eps=1e-12)
    _ok("pool_scales_l2", name, PM.check("pool_l2", outl, lref, lbound))


# --------------------------------------------------------------------------- row L2 and fp16 copies
@pytest.mark.parametrize("D", [1, 7, 256, 257, 1000, 2048, 3072])
@pytest.mark.parametrize("eps", [1e-12, 0.0])
def test_l2_normalize(D, eps):
    """Norms from 2^-60 to 2^62 (the documented range), eps-clamped rows, zero rows (0 with eps > 0, NaN with eps 0),
    out16 == out.half()."""
    ops = _ops()
    r = np.random.RandomState(D)
    x = r.standard_normal((9, D))
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x *= np.array([1, 2.0 ** -60, 2.0 ** 62, 1e-13, 0, 300, 1e-3, 1, 2.0 ** -20])[:, None]
    x[7, ::2] = 0
    xt = _t(x.astype(np.float32))
    out, o16 = ops.l2_normalize(xt, eps=eps, want_f16=True)
    torch.cuda.synchronize()
    ref, bound = PM.l2_ref(xt, eps=eps)
    _ok("l2_normalize", "D%d eps%g" % (D, eps), PM.check("l2", out, ref, bound))
    assert PM.half_bits_equal(o16, out)
    assert bool((out[4] == 0).all()) if eps > 0 else bool(torch.isnan(out[4]).all())


def _f16_specials():
    v = [0.0, -0.0, 65504.0, -65504.0, 65519.996, 65520.0, -65520.0, float("inf"), -float("inf"), float("nan"),
         2.0 ** -24, 2.0 ** -25, 2.0 ** -25 * 1.0000001, 2.0 ** -26, 3 * 2.0 ** -25, 2.0 ** -14, 2.0 ** -14 - 2.0 ** -25,
         1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 2.0 ** -11 + 2.0 ** -23, 2048 + 1.0, 2048 + 3.0, 1e-8, -1e-8]
    r = np.random.RandomState(0)
    ties = (r.randint(1024, 2048, 64) * 2 + 1).astype(np.float64) * 2.0 ** r.randint(-25, 5, 64) / 2   # odd / 2: exact ties
    sub = r.uniform(-2.0 ** -14, 2.0 ** -14, 64)
    return np.concatenate([np.array(v), ties, sub]).astype(np.float32)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 4 * 100003 + 3])
def test_f32_to_f16_equals_half(n):
    """Round to nearest even everywhere: +-0, subnormals, exact ties, 65504, 65520 -> inf, +-inf, NaN, and the n % 4
    tail after the float4 groups."""
    ops = _ops()
    sp = _f16_specials()
    r = np.random.RandomState(n)
    x = (r.standard_normal(n) * 2.0 ** r.randint(-30, 17, n)).astype(np.float32)
    x[-min(n, sp.size):] = sp[:min(n, sp.size)]
    xt = _t(x)
    for v in (xt, xt[:-1] if n > 1 else xt):
        v = v.contiguous()
        h = ops.f32_to_f16(v)
        torch.cuda.synchronize()
        assert PM.half_bits_equal(h, v), n


# --------------------------------------------------------------------------- alpha-QE
@pytest.mark.parametrize("k", [1, 2, 10, 100, 1024])
@pytest.mark.parametrize("alpha", [0.0, 0.5, 1.0, 3.0])
@pytest.mark.parametrize("D", [48, 2048])
def test_aqe(k, alpha, D):
    """Full and partial (uneven and empty shards, summed) alpha-QE with -1 entries; weights fl32(pow(s, alpha))."""
    ops = _ops()
    r = np.random.RandomState(k + D)
    Q, N = 6, 1500
    q = r.standard_normal((Q, D)).astype(np.float32)
    db = r.standard_normal((N, D)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    db /= np.linalg.norm(db, axis=1, keepdims=True)
    idx = r.randint(0, N, (Q, k)).astype(np.int64)
    idx[:, ::7] = -1
    sc = r.uniform(0.0, 1.0, (Q, k))
    sc[:, ::5] = 0.0
    args = [_t(v) for v in (q, db, idx, sc)]
    out = ops.aqe_expand(*args, alpha)
    torch.cuda.synchronize()
    ref, bound = PM.aqe_ref(*args, alpha)
    name = "k%d a%g D%d" % (k, alpha, D)
    _ok("aqe", name, PM.check("aqe", out, ref, bound))
    cuts = [0, 1, 1, 700, N]                               # shards [0,1), [1,1) empty, [1,700), [700,N)
    tot = torch.zeros((Q, D), dtype=torch.float64, device=DEV)
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        part = ops.aqe_expand(args[0], _t(db[lo:hi]) if hi > lo else args[1][:1], args[2], args[3], alpha, partial=True,
                              row_offset=lo, n_rows=hi - lo)
        pref, pbound = PM.aqe_ref(args[0], _t(db[lo:hi]) if hi > lo else args[1][:1], args[2], args[3], alpha, partial=True,
                                  row_offset=lo, n_rows=hi - lo)
        _ok("aqe_partial", "%s [%d,%d)" % (name, lo, hi), PM.check("part", part, pref, pbound))
        tot += part.double()
    full, fbound = PM.aqe_ref(*args, alpha, partial=True, row_offset=0, n_rows=N)
    assert bool(((tot - full).abs() <= fbound * 2 + 1e-30).all())


def test_aqe_negative_scores_with_fractional_alpha_give_nan_rows():
    """sim ** alpha of the reference: a negative neighbour score with a fractional alpha is NaN, and so is the row;
    integer alpha keeps the sign; other rows are unaffected."""
    ops = _ops()
    r = np.random.RandomState(9)
    q = r.standard_normal((3, 48)).astype(np.float32)
    db = r.standard_normal((20, 48)).astype(np.float32)
    idx = np.tile(np.arange(4, dtype=np.int64), (3, 1))
    sc = np.full((3, 4), 0.5)
    sc[1, 2] = -0.25
    for alpha, nan_row in ((0.5, True), (3.0, False), (1.0, False)):
        args = [_t(v) for v in (q, db, idx, sc)]
        out = ops.aqe_expand(*args, alpha)
        torch.cuda.synchronize()
        assert bool(torch.isnan(out[1]).all()) == nan_row and bool(torch.isfinite(out[[0, 2]]).all())
        ref, bound = PM.aqe_ref(*args, alpha)
        _ok("aqe", "negative a%g" % alpha, PM.check("aqe", out, ref, bound))


# --------------------------------------------------------------------------- dense exact scores
@pytest.mark.parametrize("D", [4, 2048, 2052])
def test_scores_exact(D):
    ops = _ops()
    r = np.random.RandomState(D)
    q = r.standard_normal((13, D)).astype(np.float32)
    db = (r.standard_normal((1001, D)) * 2.0 ** r.randint(-20, 20, (1001, 1))).astype(np.float32)
    db[5] = -q[0] * np.float32(3)
    out = ops.scores_exact(_t(q), _t(db))
    torch.cuda.synchronize()
    _ok("scores_exact", "D%d" % D, PM.scores_exact_check("scores", out, _t(q), _t(db)))
