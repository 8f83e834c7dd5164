"""CPU tests of the per-element bounds of tests/post_model.py: a numpy emulation of each kernel's arithmetic, in the
kernel's order, passes its bound, and each of a list of plausible bugs fails it.  At these shapes one of them (an fp16
copy rounded toward zero) passes the relative-L2 tolerances the operator tests used before (2e-5 head and
tensor-core whitening, 1e-3 fp16 copies and center bias, 1e-5 alpha-QE)."""
import numpy as np
import pytest
import torch

import post_model as PM
from conftest import rel_l2

F32 = np.float32


def _fma(a, b, c):
    """fmaf emulated: the product is exact in fp64, one rounding of the sum (a double rounding at worst)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def _tree32(v):
    """The shuffle tree over the last axis (32 lanes): v += v[lane ^ s] for s = 16 .. 1, in fp32."""
    for s in (16, 8, 4, 2, 1):
        v = (v + v[..., np.arange(32) ^ s]).astype(F32)
    return v[..., 0]


# --------------------------------------------------------------------------- emulated kernels (mutation hooks)
def emu_l2(x, eps, mut=None):
    """l2_row_body: thread t sums squares of columns t, t+256, ... (fmaf), then the block sum; sqrtf; 1/max(n, eps)."""
    x = np.asarray(x, F32)
    n, D = x.shape
    Dp = -(-D // 256) * 256
    xs = np.zeros((n, Dp), F32)
    keep = D if mut != "l2_first256" else D // 256 * 256
    xs[:, :keep] = x[:, :keep]
    ss = np.zeros((n, 256), F32)
    for j in range(Dp // 256):
        ss = _fma(xs[:, 256 * j:256 * j + 256], xs[:, 256 * j:256 * j + 256], ss)
    warps = _tree32(ss.reshape(n, 8, 32))
    tot = _tree32(np.concatenate([warps, np.zeros((n, 24), F32)], 1))
    nrm = np.sqrt(tot).astype(F32)
    den = np.maximum(nrm, F32(eps)) if eps > 0 else nrm
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (F32(1) / den).astype(F32)
        return (x * inv[:, None]).astype(F32)


def emu_f16(x, mut=None):
    """fp32 -> fp16 round to nearest even (numpy), or a bug: toward zero / the n % 4 tail left unwritten."""
    x = np.asarray(x, F32)
    h = x.astype(np.float16)
    if mut == "rz16":
        over = np.abs(h.astype(np.float64)) > np.abs(x.astype(np.float64))
        h[over] = np.nextafter(h[over], np.float16(0))
    if mut == "tail":
        flat = h.reshape(-1)
        flat[flat.size // 4 * 4:] = 0
    return h


def emu_head(feat, pooling, p, eps, norm_features, w, b, mut=None):
    """The four phases of the head in fp32, each in the kernel's order.  feat (B, HW, C) fp16 numpy."""
    B, HW, C = feat.shape
    S = PM.head_splits(HW)
    per = -(-HW // S)
    p32, eps32 = F32(p), F32(eps)
    x = feat.astype(F32)
    partial = np.zeros((B, S, C), F32)
    for s in range(S):
        beg, end = s * per, min(HW, s * per + per)
        if mut == "lost_pixel" and s == 0:
            end -= 1
        n = end - beg
        n8 = -(-n // 8) * 8
        fill = -np.inf if pooling == "max" else 0.0
        blk = np.full((B, n8, C), fill, F32)
        blk[:, :n] = x[:, beg:end]
        if pooling == "gem":
            t = np.maximum(blk, eps32)
            t = (t * t * t).astype(F32) if p32 == 3 else np.power(t, p32).astype(F32)
            t[:, n:] = 0
        else:
            t = blk
        t = t.reshape(B, n8 // 8, 8, C)
        acc = np.full((B, 8, C), fill, F32)
        for j in range(n8 // 8):
            acc = np.maximum(acc, t[:, j]) if pooling == "max" else (acc + t[:, j]).astype(F32)
        r = acc[:, 0]
        for l in range(1, 8):
            r = np.maximum(r, acc[:, l]) if pooling == "max" else (r + acc[:, l]).astype(F32)
        partial[:, s] = r
    r = partial[:, 0]
    for s in range(1, S):
        r = np.maximum(r, partial[:, s]) if pooling == "max" else (r + partial[:, s]).astype(F32)
    if pooling == "gem":
        g = np.power((r / F32(HW)).astype(F32), F32(1.0) / p32).astype(F32)
    elif pooling == "avg":
        g = (r / F32(HW)).astype(F32)
    else:
        g = r
    if norm_features:
        g = emu_l2(g, 1e-12)
    y = g
    if w is not None:
        O = w.shape[0]
        Cp = -(-C // 128) * 128
        gp = np.zeros((B, Cp), F32)
        gp[:, :C] = g
        wp = np.zeros((O, Cp), F32)
        wp[:, :C] = w
        acc = np.zeros((B, O, 32), F32)
        for j in range(Cp // 128):
            for e in range(4):
                cols = 128 * j + 4 * np.arange(32) + e
                acc = _fma(wp[None, :, cols], gp[:, None, cols], acc)
        v = _tree32(acc)
        bias = b.copy()
        if mut == "bias_last_group":
            bias[O // 8 * 8:] = 0
        y = (v + bias[None]).astype(F32)
    desc = emu_l2(y, 1e-12, "l2_first256" if mut == "l2_first256" else None)
    return dict(partial=partial, g=g, y=y, desc=desc, desc16=emu_f16(desc, mut if mut in ("rz16", "tail") else None))


def _trunc32(v):
    r = v.astype(F32)
    over = np.abs(r.astype(np.float64)) > np.abs(v)
    r[over] = np.nextafter(r[over], F32(0))
    return r


def emu_whiten_tc(x, comp, mean, cs, mut=None):
    """whiten_tc: prescaled hi/lo splits, k16 steps of (hi, lo), (lo, hi), (hi, hi), each truncated to fp32, then
    * cs.  drop_cross: both cross terms of one 64-wide K block skipped in tile (rows 0..127, cols 0..127);
    cs_shift: the last partial column tile reads the column scale one to the right."""
    hx, lx, hc, lc, csx = (t.numpy() for t in PM.whiten_tc_parts(torch.from_numpy(x), torch.from_numpy(comp),
                                                                  torch.from_numpy(mean), torch.from_numpy(cs)))
    N, D = hx.shape
    acc = np.zeros((N, hc.shape[0]), F32)
    for A, Bm, cross in ((hx, lc, True), (lx, hc, True), (hx, hc, False)):
        for k in range(D // 16):
            part = A[:, 16 * k:16 * k + 16] @ Bm[:, 16 * k:16 * k + 16].T
            if mut == "drop_cross" and cross and k // 4 == 5:
                part[:128, :128] = 0
            acc = _trunc32(acc.astype(np.float64) + part)
    c = csx.astype(F32)
    if mut == "cs_shift":
        Dout = c.shape[0]
        j0 = Dout // 128 * 128
        c = c.copy()
        c[j0:Dout - 1] = c[j0 + 1:]
    return (acc * c[None]).astype(F32)


def emu_center_bias(x16, b, mut=None):
    """center_bias_kernel in fp32; align_false: align_corners=False sampling; swap: H and W exchanged."""
    B, H, W, C = x16.shape

    def axis(i, n):
        if mut == "align_false":
            src = np.maximum((i + F32(0.5)) * F32(4.0 / n) - F32(0.5), F32(0))
        else:
            scale = F32(3.0 / (n - 1)) if n > 1 else F32(0)
            src = (scale * i.astype(F32)).astype(F32)
        i0 = np.minimum(src.astype(np.int64), 3)
        i1 = i0 + (i0 < 3)
        l1 = (src - i0).astype(F32)
        return i0, i1, (F32(1) - l1).astype(F32), l1

    nh, nw = (W, H) if mut == "swap" else (H, W)
    h0, h1, lh0, lh1 = axis(np.arange(H), nh)
    w0, w1, lw0, lw1 = axis(np.arange(W), nw)
    tab = lambda r, c: np.where(((r == 1) | (r == 2))[:, None] & ((c == 1) | (c == 2))[None, :], F32(b), F32(0))  # noqa: E731
    m = (F32(1) + (lh0[:, None] * (lw0[None] * tab(h0, w0) + lw1[None] * tab(h0, w1)) +
                   lh1[:, None] * (lw0[None] * tab(h1, w0) + lw1[None] * tab(h1, w1)))).astype(F32)
    return (x16.astype(F32) * m[None, :, :, None]).astype(np.float16)


def emu_aqe(q, db, idx, sc, alpha, mut=None):
    Q, D = q.shape
    w = np.where(idx >= 0, np.power(sc, alpha), 0).astype(F32)
    acc = q.astype(F32).copy()
    for j in range(idx.shape[1]):
        if mut == "skip" and j == 3:
            continue
        rows = db[np.maximum(idx[:, j], 0)]
        acc = np.where((idx[:, j] >= 0)[:, None], _fma(rows, w[:, j:j + 1], acc), acc)
    return emu_l2(acc, 0.0)


# --------------------------------------------------------------------------- data
def _head_case(seed=0, B=9, HW=200, C=520, O=100):
    r = np.random.RandomState(seed)
    feat = np.abs(r.standard_normal((B, HW, C))).astype(np.float16)
    feat[0, :, 3] = 0                                     # a whole zero channel: clamp to eps
    feat[1, :5, :] = np.float16(3e-6)                     # fp16 subnormals
    w = (r.standard_normal((O, C)) / np.sqrt(C)).astype(F32)
    b = (0.01 * r.standard_normal(O)).astype(F32)
    return feat, w, b


def _head_bounds(feat, w, b, pooling="gem", p=3.0, nf=False):
    t = torch.from_numpy(feat)
    return PM.head_e2e(t, pooling, p, 1e-6, nf, torch.from_numpy(w) if w is not None else None,
                       torch.from_numpy(b) if b is not None else None)


@pytest.mark.parametrize("pooling,p,nf", [("gem", 3.0, False), ("gem", 3.0000002, True), ("max", 3.0, False),
                                          ("avg", 3.0, False)])
def test_emulated_head_passes_every_phase_and_end_to_end(pooling, p, nf):
    feat, w, b = _head_case()
    out = emu_head(feat, pooling, p, 1e-6, nf, w, b)
    P, eP = PM.head_partial_ref(torch.from_numpy(feat), pooling, p, 1e-6)
    assert PM.check("partial", torch.from_numpy(out["partial"]), P, eP).ok
    g, eg = PM.head_pool_final_ref(torch.from_numpy(out["partial"]), feat.shape[1], pooling, p, nf)
    assert PM.check("g", torch.from_numpy(out["g"]), g, eg).ok
    y, ey = PM.head_fc_ref(torch.from_numpy(out["g"]), w, b)
    assert PM.check("y", torch.from_numpy(out["y"]), y, ey).ok
    d, ed = PM.l2_ref(torch.from_numpy(out["y"]), eps=1e-12)
    assert PM.check("desc", torch.from_numpy(out["desc"]), d, ed).ok
    ref, bound = _head_bounds(feat, w, b, pooling, p, nf)
    c = PM.check("e2e", torch.from_numpy(out["desc"]), ref, bound)
    assert c.ok, c.worst
    assert PM.half_bits_equal(torch.from_numpy(out["desc16"]), torch.from_numpy(out["desc"]))


def test_head_layout_matches_the_library_workspace_size():
    from dirb200 import lib
    for B, HW, C, O in [(1, 1, 512, 512), (9, 65, 520, 1000), (64, 4096, 2048, 3072), (7, 63, 2048, 128)]:
        assert PM.head_layout(B, HW, C, O)["total"] == lib.raw("dirb200_head_workspace_floats")(B, HW, C, O)


def test_emulated_kernels_pass_their_bounds():
    r = np.random.RandomState(3)
    # whitening, tensor-core path
    x = r.standard_normal((256, 2048)).astype(F32)
    mean = (0.3 * r.standard_normal(2048)).astype(F32)
    comp = (r.standard_normal((200, 2048)) / 45).astype(F32)
    cs = r.uniform(0.5, 3, 200).astype(F32)
    ref, bound, _ = PM.whiten_tc_ref(*(torch.from_numpy(v) for v in (x, comp, mean, cs)), kappa=3 * 2048 // 16)
    c = PM.check("whiten_tc", torch.from_numpy(emu_whiten_tc(x, comp, mean, cs)), ref, bound)
    assert c.ok, c.worst
    # the split itself: e' within split_error_bound of the fp32 operands' exact product
    hx, lx, hc, lc, csx = PM.whiten_tc_parts(*(torch.from_numpy(v) for v in (x, comp, mean)))
    a = torch.from_numpy(x - mean).double()
    ex = a @ torch.from_numpy(comp).double().T
    approx = (hx @ lc.T + lx @ hc.T + hx @ hc.T) * csx
    assert bool(((approx - ex).abs() <= PM.split_error_bound(*(torch.from_numpy(v) for v in (x, comp, mean)))).all())
    # SIMT whitening: fmaf chain in K order
    xs, cps = x[:10, :48], comp[:7, :48]
    acc = np.zeros((10, 7), F32)
    for k in range(48):
        acc = _fma((xs - mean[:48])[:, k:k + 1].astype(F32), cps[None, :, k], acc)
    ref, bound = PM.whiten_simt_ref(torch.from_numpy(xs), torch.from_numpy(cps), torch.from_numpy(mean[:48]), torch.from_numpy(cs[:7]))
    assert PM.check("simt", torch.from_numpy((acc * cs[:7]).astype(F32)), ref, bound).ok
    # l2, with rows at both ends of the documented range and zero rows
    v = r.standard_normal((6, 1000)).astype(F32)
    v[1] *= F32(2.0 ** -60)
    v[2] *= F32(2.0 ** 58)
    v[3] = 0
    for eps in (1e-12, 0.0):
        ref, bound = PM.l2_ref(torch.from_numpy(v), eps=eps)
        assert PM.check("l2", torch.from_numpy(emu_l2(v, eps)), ref, bound).ok
    # center bias
    xc = np.abs(r.standard_normal((2, 7, 12, 16))).astype(np.float16)
    assert PM.center_bias_check("cb", torch.from_numpy(emu_center_bias(xc, 1.5)), torch.from_numpy(xc), 1.5).ok
    # alpha-QE
    q = r.standard_normal((5, 48)).astype(F32)
    db = r.standard_normal((40, 48)).astype(F32)
    idx = r.randint(-1, 40, (5, 10)).astype(np.int64)
    sc = r.uniform(0, 1, (5, 10))
    ref, bound = PM.aqe_ref(torch.from_numpy(q), torch.from_numpy(db), torch.from_numpy(idx), torch.from_numpy(sc), 3.0)
    assert PM.check("aqe", torch.from_numpy(emu_aqe(q, db, idx, sc, 3.0)), ref, bound).ok


def test_signed_power_pool_bound_survives_zero_crossings():
    """sympow(., 1/3) near a zero crossing of the mean: a fixed tolerance would need ~1e-2, the interval bound adapts."""
    r = np.random.RandomState(5)
    a = r.standard_normal((4, 257)).astype(F32)
    b = (-a + F32(1e-7) * r.standard_normal((4, 257))).astype(F32)
    c = np.zeros_like(a)
    xs = [torch.from_numpy(v) for v in (a, b, c)]
    t = [np.sign(v) * np.power(np.maximum(np.abs(v), F32(1e-6)), F32(3)).astype(F32) for v in (a, b, c)]
    acc = ((t[0] + t[1]).astype(F32) + t[2]).astype(F32) / F32(3)
    out = np.sign(acc) * np.power(np.maximum(np.abs(acc), F32(1e-6)), F32(1) / F32(3)).astype(F32)
    ref, bound = PM.pool_scales_ref(xs, "gem", 3.0)
    assert PM.check("pool", torch.from_numpy(out.astype(F32)), ref, bound).ok
    assert float(bound.max()) > 1e-3 and float(bound.min()) < 1e-8


# --------------------------------------------------------------------------- mutations
def _mutation_outcomes():
    """name -> (fails the element bound, passes the old rel-L2 tolerance)."""
    out = {}
    feat, w, b = _head_case(seed=1, B=9, HW=200, C=1000, O=100)
    ref, bound = _head_bounds(feat, w, b)
    for mut in ("lost_pixel", "bias_last_group", "l2_first256"):
        d = emu_head(feat, "gem", 3.0, 1e-6, False, w, b, mut)["desc"]
        out[mut] = (not PM.check(mut, torch.from_numpy(d), ref, bound).ok, rel_l2(d, ref.numpy()) < PM.OLD_TOL["head"])
    good = emu_head(feat, "gem", 3.0, 1e-6, False, w, b)["desc"]
    good, ref = good[:, :99].copy(), ref[:, :99]             # 891 elements: a tail of 3 after the float4 groups
    for mut in ("rz16", "tail"):
        h = emu_f16(good, mut)
        out[mut] = (not PM.half_bits_equal(torch.from_numpy(h), torch.from_numpy(good)),
                    rel_l2(h.astype(np.float64), ref.numpy()) < PM.OLD_TOL["copy16"])
    r = np.random.RandomState(4)
    x = r.standard_normal((256, 2048)).astype(F32)
    mean = (0.3 * r.standard_normal(2048)).astype(F32)
    comp = (r.standard_normal((200, 2048)) / 45).astype(F32)
    cs = r.uniform(0.5, 3, 200).astype(F32)
    ref, bound, _ = PM.whiten_tc_ref(*(torch.from_numpy(v) for v in (x, comp, mean, cs)), kappa=PM.KAPPA_W)
    true = ((x.astype(np.float64) - mean) @ comp.astype(np.float64).T) * cs
    for mut in ("drop_cross", "cs_shift"):
        y = emu_whiten_tc(x, comp, mean, cs, mut)
        out[mut] = (not PM.check(mut, torch.from_numpy(y), ref, bound).ok, rel_l2(y, true) < PM.OLD_TOL["whiten"])
    xc = np.abs(r.standard_normal((2, 7, 12, 64))).astype(np.float16)
    exact = xc.astype(np.float64) * PM.center_bias_map64(1.0, 7, 12).numpy()[None, :, :, None]
    for mut in ("align_false", "swap"):
        y = emu_center_bias(xc, 1.0, mut)
        out[mut] = (not PM.center_bias_check(mut, torch.from_numpy(y), torch.from_numpy(xc), 1.0).ok,
                    rel_l2(y.astype(np.float64), exact) < PM.OLD_TOL["copy16"])
    q = PM.l2_ref(torch.from_numpy(r.standard_normal((8, 2048)).astype(F32)))[0].float().numpy()
    db = PM.l2_ref(torch.from_numpy(r.standard_normal((300, 2048)).astype(F32)))[0].float().numpy()
    idx = np.argsort(-(q @ db.T), axis=1)[:, :10].astype(np.int64)
    sc = np.take_along_axis(q.astype(np.float64) @ db.T.astype(np.float64), idx, 1)
    ref, bound = PM.aqe_ref(*(torch.from_numpy(v) for v in (q, db, idx, sc)), 3.0)
    y = emu_aqe(q, db, idx, sc, 3.0, "skip")
    out["aqe_skip"] = (not PM.check("aqe", torch.from_numpy(y), ref, bound).ok, rel_l2(y, ref.numpy()) < PM.OLD_TOL["aqe"])
    return out


OLD_TOLERANCE_MISSES = {"rz16"}


def test_every_mutation_fails_its_bound():
    res = _mutation_outcomes()
    print("MUTATIONS " + ", ".join("%s: bound %s, old tolerance %s" % (k, "fails" if f else "PASSES", "passes" if o else "fails")
                                   for k, (f, o) in res.items()))
    assert all(f for f, _ in res.values()), {k: v for k, v in res.items() if not v[0]}
    assert {k for k, (_, o) in res.items() if o} == OLD_TOLERANCE_MISSES
