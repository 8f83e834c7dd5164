"""fp64 references of the kernels between the layer4 map and the rows the index searches, and the per-element bounds
their outputs are held to: the head's four phases, ``center_bias``, whitening (SIMT and tensor-core paths), scale
pooling, row L2, alpha-QE and the dense exact scores.

Every check takes the exact operands the kernel saw (teacher forcing: the previous phase's GPU output where there is
one) and derives the bound from the kernel's own arithmetic.  The library builds without ``--use_fast_math``, so fp32
division and ``sqrtf`` are IEEE, FMA contraction is on, ``powf`` is within 4 ulp and the double ``pow`` within 2 ulp
(CUDA Math API tables).  ``u = 2^-24`` and ``gamma(n) = n u / (1 - n u)`` bound n fp32 roundings in a chain.  Each
reference function returns ``(ref, bound)``; the ``e_*`` arguments carry an uncertainty of the inputs, which is how the
end-to-end head bound from the fp16 layer4 map is built (``head_e2e``).

Only ``whiten_tc`` truncates (wgmma fp32 accumulation): it is held to ``KAPPA_W * 2^-23 * sum |terms|`` over its
3 D / 16 k16 steps, KAPPA_W capped at that step count, the rigorous one-truncation-per-step value.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F

F64 = torch.float64
U = 2.0 ** -24                 # fp32 unit roundoff
U64 = 2.0 ** -53
POWF_ULP = 4                   # powf, CUDA Math API (no fast math)
POW_ULP = 2                    # pow (double)
KAPPA_W = 9.89                 # 2 x 4.94, the largest accumulation ratio of whiten_tc measured on the H100 (DESIGN section 2)
HEAD_PX_LANES = 8
OLD_TOL = dict(head=2e-5, whiten=2e-5, copy16=1e-3, aqe=1e-5)   # the rel-L2 bars the operator tests used before


def gamma(n, u=U):
    if not isinstance(n, torch.Tensor):
        n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def f32(x):
    """Round to fp32 and back (fp64 tensor or float)."""
    if isinstance(x, torch.Tensor):
        return x.float().to(F64)
    return float(np.float32(x))


def ulp32(v: torch.Tensor) -> torch.Tensor:
    a = v.abs().to(F64)
    _, ex = torch.frexp(a)
    u = torch.ldexp(torch.ones_like(a), (ex - 24).to(torch.int32))
    return torch.where(a < 2.0 ** -126, torch.full_like(a, 2.0 ** -149), u)


def ulp16(v: torch.Tensor) -> torch.Tensor:
    a = v.abs().to(F64)
    _, ex = torch.frexp(a)
    u = torch.ldexp(torch.ones_like(a), (ex - 11).to(torch.int32))
    return torch.where(a < 2.0 ** -14, torch.full_like(a, 2.0 ** -24), u)


# --------------------------------------------------------------------------- outcome of a check
@dataclass
class Check:
    """n elements, n_fail outside the bound (NaN where the reference is finite, or the reverse, fails), ratio = the
    largest |gpu - ref| / bound, and the worst failing element."""
    name: str
    n: int
    n_fail: int
    ratio: float
    worst: str = ""

    @property
    def ok(self):
        return self.n_fail == 0


def check(name, got, ref, bound) -> Check:
    g = torch.as_tensor(got).to(device=ref.device, dtype=F64)
    ref = ref.to(F64)
    bound = torch.as_tensor(bound, dtype=F64, device=ref.device).expand_as(ref)
    nan_r, nan_g = torch.isnan(ref), torch.isnan(g)
    d = (g - ref).abs()
    d = torch.where(nan_r & nan_g, torch.zeros_like(d), d)
    same_inf = torch.isinf(ref) & (g == ref)
    d = torch.where(same_inf, torch.zeros_like(d), d)
    bad = ~(d <= bound) | (nan_r != nan_g)
    ratio = torch.where(bound > 0, d / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(d > 0, torch.full_like(d, math.inf), torch.zeros_like(d)))
    n_fail = int(bad.sum())
    worst = ""
    if n_fail:
        flat = torch.nonzero(bad.reshape(-1)).reshape(-1)
        i = int(flat[torch.argmax(torch.nan_to_num(d.reshape(-1)[flat], nan=math.inf))])
        idx = np.unravel_index(i, tuple(ref.shape))
        worst = "worst failing element %s: gpu %.9g ref %.9g bound %.3g" % (
            tuple(int(v) for v in idx), float(g.reshape(-1)[i]), float(ref.reshape(-1)[i]), float(bound.reshape(-1)[i]))
    r = torch.nan_to_num(ratio, nan=math.inf)
    return Check(name, ref.numel(), n_fail, float(r.max()) if r.numel() else 0.0, worst)


def half_bits_equal(h16: torch.Tensor, x32: torch.Tensor) -> bool:
    """fp16 copy == x32.half() bit for bit (any NaN matches any NaN)."""
    want = x32.half()
    a, b = h16.reshape(-1), want.reshape(-1)
    nan_a, nan_b = torch.isnan(a), torch.isnan(b)
    if not torch.equal(nan_a, nan_b):
        return False
    return torch.equal(a[~nan_a].view(torch.int16), b[~nan_b].view(torch.int16))


# --------------------------------------------------------------------------- row L2 (l2_row_body, pool_scales, aqe)
def l2_depth(D):
    """Roundings of the block sum of squares: ceil(D/256) per thread (the square folds into an FMA), 5 shuffle steps,
    5 more over the warp partials."""
    return -(-D // 256) + 10


def l2_ref(x, e=None, eps=0.0, depth=None):
    """out = x / max(||x||, eps) (eps 0: x / ||x||, NaN for a zero row) for GPU input x~ within e of x.  The kernel:
    ss = fp32 sum of squares (gamma(depth + 1), plus 2^-149 per entry for squares in the subnormal range), sqrtf,
    1 / max(nrm, eps), one multiply.  Holds for 2^-63 <~ ||x|| <~ 2^64: below, the squares underflow (a row is then far
    below any eps > 0 and comes out x / eps as the reference); above, ss overflows to inf and the row comes out 0."""
    x = x.to(F64)
    D = x.shape[-1]
    e = torch.zeros_like(x) if e is None else e.to(F64)
    depth = l2_depth(D) if depth is None else depth
    N = torch.linalg.vector_norm(x, dim=-1, keepdim=True)
    E = torch.linalg.vector_norm(e, dim=-1, keepdim=True)
    den = torch.clamp(N, min=eps) if eps > 0 else N
    ref = x / den
    lo = torch.clamp(N - E, min=0.0)
    ss_rel = float(gamma(depth + 1)) + D * 2.0 ** -149 / torch.where(lo > 0, lo * lo, torch.ones_like(lo))
    dn = 0.5 * ss_rel * 1.01 + U
    rho = (N * dn + E * (1 + dn)) / torch.where(den > 0, den, torch.ones_like(den))
    rho = torch.where(lo > 0, rho, torch.where(den > 0, rho, torch.full_like(rho, math.inf)))
    scale = 1.0 / (torch.where(den > 0, den, torch.ones_like(den)) * torch.clamp(1 - rho, min=1e-300))
    bound = (e + x.abs() * rho) * scale + 2.1 * U * (x.abs() + e) * scale
    bound = torch.where(rho < 0.5, bound, torch.full_like(bound, math.inf))
    return ref, bound


# --------------------------------------------------------------------------- head (ops.cu:89-442)
def head_splits(hw):
    return max(1, min(16, hw // 64))


def _align32(n):
    return (n + 31) // 32 * 32


def head_layout(B, HW, C, out_dim):
    """Offsets (floats) of partial, g, y in the workspace of head_pool_fc_l2, and its total size, as ops.cu lays them."""
    S = head_splits(HW)
    o_g = _align32(B * S * C)
    o_y = o_g + _align32(B * C)
    total = o_y + _align32(B * max(out_dim, C)) + 32
    return dict(S=S, partial=0, g=o_g, y=o_y, total=total)


def _term_rel(p32):
    """Relative error of one GeM term: x*x*x (two roundings) for p = 3, else powf."""
    return float(gamma(2)) if p32 == 3.0 else POWF_ULP * 2.0 ** -23


def head_partial_ref(feat, pooling, p, eps, e_in=None):
    """Phase 1: partial[b][s][c] over the pixels [s*per, min(HW, (s+1)*per)) of split s, per = ceil(HW/S).  Each of the
    8 pixel lanes sums its pixels in order, then the 8 lane sums are added: ceil(n/8) + 7 roundings.  GeM terms
    max(x, eps)^p; max pooling exact.  feat (B, HW, C) fp16 values; e_in: their uncertainty (end-to-end bound)."""
    B, HW, C = feat.shape
    S = head_splits(HW)
    per = -(-HW // S)
    x = feat.to(F64)
    pad = S * per - HW
    valid = torch.ones(B, HW, 1, dtype=torch.bool, device=x.device)
    if pad:
        x = F.pad(x, (0, 0, 0, pad))
        valid = F.pad(valid, (0, 0, 0, pad))
    e = None
    if e_in is not None:
        e = F.pad(e_in.to(F64), (0, 0, 0, pad)) if pad else e_in.to(F64)
    x, valid = x.reshape(B, S, per, C), valid.reshape(B, S, per, 1)
    e = e.reshape(B, S, per, C) if e is not None else None
    counts = valid.sum(2).to(F64)                                            # (B, S, 1)
    depth = torch.ceil(counts / HEAD_PX_LANES) + HEAD_PX_LANES - 1
    if pooling == "max":
        ref = torch.where(valid, x, torch.full_like(x, -math.inf)).amax(2)
        bound = torch.zeros_like(ref) if e is None else torch.where(valid, e, torch.zeros_like(e)).amax(2)
        return ref, bound
    p32, eps32 = f32(p), f32(eps)
    if pooling == "gem":
        t = torch.clamp(x, min=eps32) ** p32
        rel = _term_rel(p32)
        dt = torch.zeros_like(t)
        if e is not None:
            hi = torch.clamp(x + e, min=eps32) ** p32
            lo = torch.clamp(x - e, min=eps32) ** p32
            dt = torch.maximum(hi - t, t - lo)
    else:
        t, rel = x, 0.0
        dt = torch.zeros_like(t) if e is None else e
    t = torch.where(valid, t, torch.zeros_like(t))
    dt = torch.where(valid, dt, torch.zeros_like(dt))
    ref = t.sum(2)
    m = t.abs().sum(2) + dt.sum(2)
    bound = dt.sum(2) + m * rel + gamma(depth) * m * (1 + rel)
    return ref, bound


def head_pool_final_ref(partial, HW, pooling, p, norm_features=False, e_part=None):
    """Phase 2: the Sb partial sums added in order (Sb - 1 roundings), / HW, then powf(., fl32(1/p)) for GeM; the
    reference exponent is 1/p exactly, so the fl32(1/p) - 1/p difference is part of the bound.  GeM is bounded by
    evaluating the reference at both ends of the interval of the mean (the map is monotone), widened by powf's 4 ulp.
    norm_features: then the L2 over channels (eps 1e-12, depth from C)."""
    P = partial.to(F64)
    S = P.shape[1]
    ep = torch.zeros_like(P) if e_part is None else e_part.to(F64)
    if pooling == "max":
        ref, bound = P.amax(1), ep.amax(1)
    else:
        R = P.sum(1)
        eR = ep.sum(1) + float(gamma(S - 1)) * (P.abs().sum(1) + ep.sum(1))
        if pooling == "avg":
            ref = R / HW
            bound = eR / HW + U * (R.abs() + eR) / HW
        else:
            p32 = f32(p)
            q, q32 = 1.0 / p32, f32(1.0 / p32)
            ref = (R / HW) ** q
            lo = torch.clamp((R - eR) / HW * (1 - U), min=0.0)
            hi = (R + eR) / HW * (1 + U)
            top = torch.maximum(hi ** q, hi ** q32) * (1 + POWF_ULP * 2.0 ** -23)
            bot = torch.minimum(lo ** q, lo ** q32) * (1 - POWF_ULP * 2.0 ** -23)
            bound = torch.maximum(top - ref, ref - bot)
    if norm_features:
        ref, bound = l2_ref(ref, bound, eps=1e-12, depth=l2_depth(ref.shape[-1]))
    return ref, bound


def fc_depth(C):
    """Roundings of one FC output: 4 fmaf per float4 group, ceil(C/128) groups per lane, 5 shuffle steps, + bias."""
    return 4 * -(-C // 128) + 6


def head_fc_ref(g, w, b, e_g=None):
    """Phase 3: y = g W^T + bias, held to gamma(fc_depth) * (sum |W||g| + |b|) (+ the propagated input error)."""
    g = g.to(F64)
    w = torch.as_tensor(w).to(device=g.device, dtype=F64)
    b = torch.zeros(w.shape[0], dtype=F64, device=g.device) if b is None else torch.as_tensor(b).to(device=g.device, dtype=F64)
    ref = g @ w.T + b
    prop = torch.zeros_like(ref) if e_g is None else e_g.to(F64) @ w.abs().T
    m = g.abs() @ w.abs().T + b.abs() + prop
    return ref, prop + gamma(fc_depth(g.shape[1])) * m


def head_e2e(feat, pooling, p, eps, norm_features, fc_w, fc_b, e_in=None):
    """The head's bound from its fp16 input to the L2-normalised descriptor: every phase's bound propagated through
    the next (no GPU intermediate is read)."""
    HW = feat.shape[1]
    P, eP = head_partial_ref(feat, pooling, p, eps, e_in)
    g, eg = head_pool_final_ref(P, HW, pooling, p, norm_features, eP)
    if fc_w is not None:
        g, eg = head_fc_ref(g, fc_w, fc_b, eg)
    return l2_ref(g, eg, eps=1e-12)


# --------------------------------------------------------------------------- center_bias (ops.cu:486-540)
def center_bias_map64(b, H, W, device=None):
    """1 + bilinear(align_corners=True) of the 4x4 map with b on its central 2x2, in fp64 (O.center_bias_map)."""
    from oracle import dir_oracle as O
    return O.center_bias_map(b, H, W, dtype=F64).to(device)[0, 0]


def center_bias_ref(x16, b):
    """x (B, H, W, C) fp16 -> fl16(x * m).  The kernel forms m in fp32 (a few roundings on terms <= b): allow 16 ulp32 of
    m times |x| plus half an fp16 ulp of the result."""
    x = x16.to(F64)
    m = center_bias_map64(b, x.shape[1], x.shape[2], x.device)[None, :, :, None]
    ref = x * m
    return ref, x.abs() * m * 16 * U


def center_bias_check(name, y16, x16, b):
    ref, b1 = center_bias_ref(x16, b)
    y = y16.to(F64).to(ref.device)
    return check(name, y, ref, b1 + 0.5 * ulp16(torch.maximum(y.abs(), ref.abs())))


# --------------------------------------------------------------------------- whitening (ops.cu:615-856)
def centred(x32, mean32):
    """fl32(x - mean), the kernel's first operation (IEEE subtraction in fp32)."""
    return x32.float() if mean32 is None else (x32.float() - mean32.float())


def whiten_simt_ref(x32, comp32, mean32=None, cs32=None):
    """whiten_gemm_kernel: an fmaf chain over K in order (D roundings), then * colscale."""
    a = centred(x32, mean32).to(F64)
    c = comp32.to(device=a.device, dtype=F64)
    D = a.shape[1]
    e, m = a @ c.T, a.abs() @ c.abs().T
    cs = torch.ones(c.shape[0], dtype=F64, device=a.device) if cs32 is None else cs32.to(device=a.device, dtype=F64)
    ref = e * cs
    bound = cs.abs() * (float(gamma(D)) + float(gamma(D, U64))) * m * (1 + U) + U * ref.abs()
    return ref, bound


def prescale(absmax: float) -> float:
    """prescale_for: the power of two that puts absmax in [2^13, 2^14), shift clamped to +-40; 1 for 0."""
    if not absmax > 0:
        return 1.0
    _, e = math.frexp(absmax)
    return 2.0 ** max(-40, min(40, 14 - e))


def split16(v32: torch.Tensor, s: float):
    """split_f16_kernel: v * s (exact), hi = fl16, lo = fl16(v*s - hi) (the difference is exact in fp32)."""
    vs = v32.float() * s
    hi = vs.half()
    lo = (vs - hi.float()).half()
    return hi.to(F64), lo.to(F64)


def whiten_tc_parts(x32, comp32, mean32=None, cs32=None):
    """The tensor-core path's operands: prescales from the global absmax of x - mean and of comp, hi/lo splits, and the
    column scale cs = fl32(colscale * fl32(1 / (sx * sc))).  -> (hx, lx, hc, lc, cs)."""
    a = centred(x32, mean32)
    c = comp32.float().to(a.device)
    fin = lambda t: float(t.abs()[torch.isfinite(t)].max()) if t.numel() else 0.0   # noqa: E731
    sx, sc = prescale(fin(a)), prescale(fin(c))
    hx, lx = split16(a, sx)
    hc, lc = split16(c, sc)
    inv = f32(1.0 / f32(sx * sc))
    cs = torch.ones(c.shape[0], dtype=torch.float32, device=a.device) if cs32 is None else cs32.float().to(a.device)
    return hx, lx, hc, lc, (cs * np.float32(inv)).to(F64)


def whiten_tc_ref(x32, comp32, mean32=None, cs32=None, kappa=None):
    """whiten_tc: e' = sum (hx lc + lx hc + hx hc) (lo*lo is dropped by design) times cs; the wgmma accumulation of the
    3 D / 16 k16 steps loses at most KAPPA_W * 2^-23 * T, T = sum of the |terms|; then one fp32 multiply.
    -> (ref, bound, acc) with acc = |cs| 2^-23 T, the unit of the accumulation ratio."""
    hx, lx, hc, lc, cs = whiten_tc_parts(x32, comp32, mean32, cs32)
    D = hx.shape[1]
    kappa = min(KAPPA_W if kappa is None else kappa, 3 * D // 16)
    e = hx @ lc.T + lx @ hc.T + hx @ hc.T
    T = hx.abs() @ (hc.abs() + lc.abs()).T + lx.abs() @ hc.abs().T
    ref = e * cs
    acc = cs.abs() * 2.0 ** -23 * T
    bound = kappa * acc * (1 + U) + cs.abs() * float(gamma(3 * D, U64)) * T + U * ref.abs() * (1 + 1e-6)
    return ref, bound, acc


def split_error_bound(x32, comp32, mean32=None):
    """|sum v c - (hx lc + lx hc + hx hc) / (sx sc)| element by element: lo*lo plus the rounding of the lo halves,
    2^-22 relative per operand with an absolute 2^-25 floor (fp16 subnormals) in scaled units."""
    a = centred(x32, mean32)
    c = comp32.float().to(a.device)
    fin = lambda t: float(t.abs()[torch.isfinite(t)].max()) if t.numel() else 0.0   # noqa: E731
    sx, sc = prescale(fin(a)), prescale(fin(c))
    hx, lx = split16(a, sx)
    hc, lc = split16(c, sc)
    va, vc = a.to(F64).abs() * sx, c.to(F64).abs() * sc
    dx, dc = 2.0 ** -22 * va + 2.0 ** -25, 2.0 ** -22 * vc + 2.0 ** -25
    return (lx.abs() @ lc.abs().T + (va + dx) @ dc.T + dx @ vc.T) / (sx * sc)


# --------------------------------------------------------------------------- scale pooling (ops.cu:550-592)
def sympow(v, q, eps):
    return torch.sign(v) * torch.clamp(v.abs(), min=eps) ** q


def pool_scales_ref(xs, pooling, gemp):
    """pool_scales_kernel before its L2: mean over S chains (S roundings, then / S), or the signed power mean
    sympow(mean(sympow(x, p)), 1/p) with the 1e-6 clamp.  sympow(., 1/p) has unbounded slope at 0, so its bound comes
    from evaluating the reference at both ends of the interval of the mean (the map is monotone), for both 1/p and the
    kernel's fl32(1/p), widened by powf's 4 ulp.  S = 1 is the identity: exact."""
    x = torch.stack([t.to(F64) for t in xs], 0)
    S = x.shape[0]
    if S == 1:
        return x[0], torch.zeros_like(x[0])
    div = U
    if pooling == "mean":
        ref = x.mean(0)
        return ref, float(gamma(S)) * x.abs().sum(0) / S + div * (ref.abs() + float(gamma(S)) * x.abs().sum(0) / S)
    p32, eps = f32(gemp), f32(1e-6)
    t = sympow(x, p32, eps)
    rel = POWF_ULP * 2.0 ** -23
    A = t.mean(0)
    EA = (rel + float(gamma(S)) * (1 + rel)) * t.abs().sum(0) / S + div * (A.abs() + t.abs().sum(0) / S * 2 * rel)
    q, q32 = 1.0 / p32, f32(1.0 / p32)
    ref = sympow(A, q, eps)
    cand = [sympow(A + s * EA, qq, eps) for s in (-1.0, 1.0) for qq in (q, q32)]
    top = torch.stack(cand).amax(0)
    bot = torch.stack(cand).amin(0)
    top = top + top.abs() * rel
    bot = bot - bot.abs() * rel
    return ref, torch.maximum(top - ref, ref - bot)


# --------------------------------------------------------------------------- alpha-QE (search.cu:493-533)
def aqe_ref(q32, db32, nn_idx, nn_scores, alpha, partial=False, row_offset=0, n_rows=0):
    """out_i = normalize(q_i + sum_j db[r_ij] * s_ij^alpha) in j order, or the un-normalised neighbour sum of this
    shard's rows (partial).  The weight is fl32(pow(s, alpha)) (2 ulp in fp64, then one fp32 rounding); each neighbour
    is one fmaf (k roundings); then 1 / sqrtf(sum of squares).  A negative score with a fractional alpha gives a NaN
    weight and a NaN row, as the reference's sim ** alpha does.  -> (ref, bound)."""
    dev = q32.device
    q = q32.to(F64)
    db = db32.to(device=dev, dtype=F64)
    idx = nn_idx.to(dev).clone()
    s = nn_scores.to(device=dev, dtype=F64)
    if partial or n_rows > 0:
        loc = idx - row_offset
        idx = torch.where((idx >= 0) & (loc >= 0) & (loc < n_rows), loc, torch.full_like(idx, -1))
    valid = idx >= 0
    w = torch.where(valid, torch.pow(s, float(alpha)), torch.zeros_like(s))
    rows = db[torch.clamp(idx, min=0)] * valid[..., None]                   # (Q, k, D)
    ref = (rows * w[..., None]).sum(1)
    m = (rows.abs() * w.abs()[..., None]).sum(1)
    if not partial:
        ref = ref + q
    mq = m + (0 if partial else q.abs())
    k = nn_idx.shape[1]
    bound = m * (U + POW_ULP * U64) * (1 + U) + float(gamma(k)) * (mq + m * 2 * U)
    if partial:
        return ref, bound
    return l2_ref(ref, bound, eps=0.0)


# --------------------------------------------------------------------------- dense exact scores (search.cu:465-491)
def scores_exact_ref(q32, db32):
    """fp64 accumulation of exact fp32 products, rounded to fp32: |out - e| <= 1/2 ulp32 + gamma64(D) sum |q r| (the
    reference's own fp64 sum counted twice)."""
    q, r = q32.to(F64), db32.to(device=q32.device, dtype=F64)
    e, m = q @ r.T, q.abs() @ r.abs().T
    return e, 2 * float(gamma(q.shape[1], U64)) * m


def scores_exact_check(name, out, q32, db32):
    e, b = scores_exact_ref(q32, db32)
    o = out.to(device=e.device, dtype=F64)
    return check(name, o, e, b + 0.5 * ulp32(torch.maximum(o.abs(), e.abs())))
